// Shading terms of point and directional lights (include/r3dg_b200.h, LIGHTS; DESIGN.md §4.26): each light is the
// shading step's one incident sample along l with visibility T, global light E and zero local light, evaluated with
// the shading step's own GGX code (brdf.cuh) and compiled with its flags (-fmad=false).
//
// Design notes
//  * one thread per Gaussian: its material, normal and mean are loaded once for all lights and views; the K lights
//    sit in shared memory; views are the outer loop, lights the inner one, so each view's sums run in one-view order
//    and every view's outputs equal a one-view call's bit for bit.
//  * the backward recomputes the forward, writes the per-Gaussian gradient rows directly (per-view sums added in view
//    order) and reduces the light gradients without atomics: per (view, light) a warp butterfly, added by lane 0 to
//    the warp's shared-memory row, the warps' rows summed in warp order into the CTA's partial [K,6], and the
//    partials summed in block order by lights_reduce_kernel.  The grid depends on P only, so every output is
//    bitwise reproducible.
#include "kernels.h"
#include "lights_eval.cuh"

namespace r3dg {

static int lights_blocks(int P) { return (P + LS_THREADS - 1) / LS_THREADS; }

__global__ void __launch_bounds__(LS_THREADS) lights_fwd_kernel(const r3dg_light_args a, const uint32_t point_mask) {
    __shared__ LightSmem s;
    stage_lights(a, s);
    const int g = blockIdx.x * LS_THREADS + threadIdx.x;
    if (g >= a.P) return;
    GaussianOperands o;
    load_material(a, g, o);
    const float m[3] = {a.means3D[3 * (size_t)g], a.means3D[3 * (size_t)g + 1], a.means3D[3 * (size_t)g + 2]};
    const float* Trow = a.shadows + (size_t)g * a.K;
    for (int v = 0; v < a.V; ++v) {
        const size_t row = (size_t)v * a.P + g;
        view_operands(o.n, a.viewdirs + 3 * row, o.V, o.vnorm, o.Ns);
        float pbr[3] = {0.f, 0.f, 0.f}, spec[3] = {0.f, 0.f, 0.f}, diff[3] = {0.f, 0.f, 0.f};
        for (int j = 0; j < a.K; ++j) {
            const LightTerm t = light_term((point_mask >> j) & 1, s, j, o, m);
            const float T = Trow[j];
            GgxEval e;
            eval_ggx<false>(o.V, o.Ns, o, t.d.l[0], t.d.l[1], t.d.l[2], e);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float tr = t.E[c] * T * t.ndi;                  // (global light * visibility) * area (1) * n.w
                const float fd = o.base[c] / PI_F;
                pbr[c] += (fd + e.fs) * tr; spec[c] += e.fs * tr; diff[c] += tr;
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) { a.pbr[3 * row + c] = pbr[c]; a.specular[3 * row + c] = spec[c]; a.diffuse_light[3 * row + c] = diff[c]; }
    }
}

// partial: [gridDim.x][K][6] = (dL/dvec, dL/dcolor) of each light summed over the CTA's Gaussians and the views
__global__ void __launch_bounds__(LS_THREADS) lights_bwd_kernel(const r3dg_light_args a, const uint32_t point_mask, float* __restrict__ partial) {
    __shared__ LightSmem s;
    __shared__ float sAcc[LS_WARPS][R3DG_MAX_LIGHTS * 6];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < LS_WARPS * R3DG_MAX_LIGHTS * 6; i += LS_THREADS) (&sAcc[0][0])[i] = 0.f;
    stage_lights(a, s);
    const int g_raw = blockIdx.x * LS_THREADS + threadIdx.x;
    const bool valid = g_raw < a.P;
    const int g = valid ? g_raw : a.P - 1;        // idle threads of the last CTA shade a copy, contribute zeros
    GaussianOperands o;
    load_material(a, g, o);
    const float m[3] = {a.means3D[3 * (size_t)g], a.means3D[3 * (size_t)g + 1], a.means3D[3 * (size_t)g + 2]};
    const float* Trow = a.shadows + (size_t)g * a.K;
    float dbase[3] = {0.f, 0.f, 0.f}, drough = 0.f, dmean[3] = {0.f, 0.f, 0.f};
    for (int v = 0; v < a.V; ++v) {
        const size_t row = (size_t)v * a.P + g;
        view_operands(o.n, a.viewdirs + 3 * row, o.V, o.vnorm, o.Ns);
        float gp[3], gs[3], gd[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            gp[c] = valid ? a.dL_dpbr[3 * row + c] : 0.f;
            gs[c] = valid && a.dL_dspecular ? a.dL_dspecular[3 * row + c] : 0.f;
            gd[c] = valid && a.dL_ddiffuse_light ? a.dL_ddiffuse_light[3 * row + c] : 0.f;
        }
        float dbase_v[3] = {0.f, 0.f, 0.f}, drough_v = 0.f, dmean_v[3] = {0.f, 0.f, 0.f}, dV[3] = {0.f, 0.f, 0.f};
        for (int j = 0; j < a.K; ++j) {
            const int kind = (point_mask >> j) & 1;
            const LightTerm t = light_term(kind, s, j, o, m);
            const float T = Trow[j];
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
            // GGX: roughness, view and the normalised direction L_n = l / max(|l|, eps) it forms from l
            float dLn[3], dl[3];
            ggx_backward<true>(o.V, o.Ns, o, e, dfs, drough_v, dV, dLn);
            LightDir ll;
            ll.l[0] = t.d.l[0]; ll.l[1] = t.d.l[1]; ll.l[2] = t.d.l[2];
            ll.rn = sqrtf(ll.l[0] * ll.l[0] + ll.l[1] * ll.l[1] + ll.l[2] * ll.l[2]);
            const float lden = fmaxf(ll.rn, LIGHT_EPS);
#pragma unroll
            for (int c = 0; c < 3; ++c) ll.l[c] = ll.l[c] / lden;
            normalize_backward(ll, dLn, dl);
            const float dn = t.ndr >= 0.f ? dndi : 0.f;                   // clamp(min=0) passes the gradient at 0
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
                for (int c = 0; c < 3; ++c) { dvc[c] = dw[c] + 2.0f * t.d.w[c] * dr2; dmean_v[c] -= dvc[c]; }
            }
            // the light's gradient: summed over the warp (fixed butterfly), added to the warp's row by lane 0
#pragma unroll
            for (int q = 0; q < 6; ++q) {
                const float x = warp_sum(valid ? dvc[q] : 0.f);
                if (lane == 0) sAcc[warp][6 * j + q] += x;
            }
        }
        if (valid) {
            const float vd = o.V[0] * dV[0] + o.V[1] * dV[1] + o.V[2] * dV[2];
#pragma unroll
            for (int c = 0; c < 3; ++c) a.dL_dviewdirs[3 * row + c] = (dV[c] - o.V[c] * vd) / o.vnorm;   // through V = normalize(viewdirs)
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) { dbase[c] += dbase_v[c]; dmean[c] += dmean_v[c]; }
        drough += drough_v;
    }
    if (valid) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { a.dL_dbase_color[3 * (size_t)g + c] = dbase[c]; a.dL_dmeans3D[3 * (size_t)g + c] = dmean[c]; }
        a.dL_droughness[g] = drough;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 6 * a.K; i += LS_THREADS) {
        float x = sAcc[0][i];
#pragma unroll
        for (int w = 1; w < LS_WARPS; ++w) x += sAcc[w][i];
        partial[(size_t)blockIdx.x * 6 * a.K + i] = x;
    }
}

// dL/dvec and dL/dcolor: one warp per (light, component), the partials summed in block order (lane-strided, then a
// fixed butterfly)
__global__ void __launch_bounds__(LS_THREADS) lights_reduce_kernel(int K, int blocks, const float* __restrict__ partial,
                                                                   float* __restrict__ dvec, float* __restrict__ dcolor) {
    const int i = blockIdx.x * LS_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= 6 * K) return;
    float x = 0.f;
    for (int b = lane; b < blocks; b += 32) x += partial[(size_t)b * 6 * K + i];
    x = warp_sum(x);
    if (lane == 0) {
        const int j = i / 6, q = i % 6;
        if (q < 3) dvec[3 * j + q] = x;
        else dcolor[3 * j + q - 3] = x;
    }
}

// ---- host launchers -----------------------------------------------------------------------
int launch_lights_reduce(int K, int blocks, const float* partial, float* dvec, float* dcolor, cudaStream_t stream) {
    lights_reduce_kernel<<<(6 * K + LS_WARPS - 1) / LS_WARPS, LS_THREADS, 0, stream>>>(K, blocks, partial, dvec, dcolor);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

size_t shade_lights_work_bytes(int P, int K) {
    return P <= 0 || K <= 0 ? 0 : (size_t)lights_blocks(P) * 6 * K * sizeof(float);
}

static bool lights_args_valid(const r3dg_light_args* a) {
    if (!a || a->P < 0 || a->V < 1 || a->V > R3DG_MAX_VIEWS || !lights_valid(a->K, a->kind)) return false;
    if (a->K > 0 && (!a->vec || !a->color)) return false;
    if (a->P > 0 && (!a->means3D || !a->base_color || !a->roughness || !a->normals || !a->viewdirs || (a->K > 0 && !a->shadows)))
        return false;
    return true;
}

int launch_shade_lights_forward(const r3dg_light_args* a, cudaStream_t stream, bool* launched) {
    *launched = false;
    if (!lights_args_valid(a)) return R3DG_ERR_BAD_ARG;
    if (a->P > 0 && (!a->pbr || !a->diffuse_light || !a->specular)) return R3DG_ERR_BAD_ARG;
    if (a->P == 0) return 0;
    if (a->K == 0) {
        const size_t n = (size_t)a->V * a->P * 3 * sizeof(float);
        R3DG_CUDA_TRY(cudaMemsetAsync(a->pbr, 0, n, stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->diffuse_light, 0, n, stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->specular, 0, n, stream));
        return 0;
    }
    lights_fwd_kernel<<<lights_blocks(a->P), LS_THREADS, 0, stream>>>(*a, point_mask(a->K, a->kind));
    R3DG_CUDA_TRY(cudaGetLastError());
    *launched = true;
    return 0;
}

int launch_shade_lights_backward(const r3dg_light_args* a, cudaStream_t stream, bool* launched) {
    *launched = false;
    if (!lights_args_valid(a)) return R3DG_ERR_BAD_ARG;
    if (a->P > 0 && (!a->dL_dpbr || !a->dL_dbase_color || !a->dL_droughness || !a->dL_dviewdirs || !a->dL_dmeans3D))
        return R3DG_ERR_BAD_ARG;
    if (a->K > 0 && (!a->dL_dvec || !a->dL_dcolor)) return R3DG_ERR_BAD_ARG;
    const size_t need = shade_lights_work_bytes(a->P, a->K);
    if (need > 0 && (!a->work || a->work_bytes < need)) return R3DG_ERR_BAD_ARG;
    if (a->P == 0 || a->K == 0) {
        if (a->P > 0) {
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dbase_color, 0, (size_t)a->P * 3 * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_droughness, 0, (size_t)a->P * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dviewdirs, 0, (size_t)a->V * a->P * 3 * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dmeans3D, 0, (size_t)a->P * 3 * sizeof(float), stream));
        }
        if (a->K > 0) {
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dvec, 0, (size_t)a->K * 3 * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dcolor, 0, (size_t)a->K * 3 * sizeof(float), stream));
        }
        return 0;
    }
    const int blocks = lights_blocks(a->P);
    float* partial = (float*)a->work;
    lights_bwd_kernel<<<blocks, LS_THREADS, 0, stream>>>(*a, point_mask(a->K, a->kind), partial);
    R3DG_CUDA_TRY(cudaGetLastError());
    const int rc = launch_lights_reduce(a->K, blocks, partial, a->dL_dvec, a->dL_dcolor, stream);
    if (rc != 0) return rc;
    *launched = true;
    return 0;
}

// ==== spot and rect lights (SHAPED LIGHTS; DESIGN.md §4.28) ==================================================
// The same layout as above: one thread per Gaussian, views outer, lights then samples inner, so every view's sums run
// in one-view order.  A rect sample's point y_q is rect_sample's (lights.cuh), bit for bit the trace's.  The backward
// accumulates each light's gradient over its samples in registers (SL_SLOTS, lights_eval.cuh), sums them over the warp
// and the CTA as lights_bwd_kernel does, and shaped_reduce_kernel sums the CTAs in block order and applies the
// light-level chain rule once (axis normalisation, u x v, n_e and A).

__global__ void __launch_bounds__(LS_THREADS) shaped_fwd_kernel(const r3dg_shaped_light_args a, const uint32_t rect_mask, const int R) {
    __shared__ ShapedSmem s;
    stage_shaped(a, rect_mask, s);
    const int g = blockIdx.x * LS_THREADS + threadIdx.x;
    if (g >= a.P) return;
    GaussianOperands o;
    load_material(a, g, o);
    const float m[3] = {a.means3D[3 * (size_t)g], a.means3D[3 * (size_t)g + 1], a.means3D[3 * (size_t)g + 2]};
    const float* Trow = a.shadows + (size_t)g * R;
    for (int v = 0; v < a.V; ++v) {
        const size_t row = (size_t)v * a.P + g;
        view_operands(o.n, a.viewdirs + 3 * row, o.V, o.vnorm, o.Ns);
        float pbr[3] = {0.f, 0.f, 0.f}, spec[3] = {0.f, 0.f, 0.f}, diff[3] = {0.f, 0.f, 0.f};
        int col = 0;
        for (int j = 0; j < a.K; ++j) {
            const bool rect = (rect_mask >> j) & 1;
            const int n = rect ? a.M * a.M : 1;
            const uint32_t h = rect_hash(a.seed, (uint32_t)g, (uint32_t)j);
            for (int q = 0; q < n; ++q, ++col) {
                ShapedTerm t;
                shaped_term(rect, s, j, a.M, h, q, o, m, t);
                const float T = Trow[col];
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
#pragma unroll
        for (int c = 0; c < 3; ++c) { a.pbr[3 * row + c] = pbr[c]; a.specular[3 * row + c] = spec[c]; a.diffuse_light[3 * row + c] = diff[c]; }
    }
}

// partial: [gridDim.x][K][SL_SLOTS], summed over the CTA's Gaussians, the views and the samples
__global__ void __launch_bounds__(LS_THREADS) shaped_bwd_kernel(const r3dg_shaped_light_args a, const uint32_t rect_mask, const int R,
                                                                float* __restrict__ partial) {
    __shared__ ShapedSmem s;
    __shared__ float sAcc[LS_WARPS][R3DG_MAX_LIGHTS * SL_SLOTS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < LS_WARPS * R3DG_MAX_LIGHTS * SL_SLOTS; i += LS_THREADS) (&sAcc[0][0])[i] = 0.f;
    stage_shaped(a, rect_mask, s);
    const int g_raw = blockIdx.x * LS_THREADS + threadIdx.x;
    const bool valid = g_raw < a.P;
    const int g = valid ? g_raw : a.P - 1;        // idle threads of the last CTA shade a copy, contribute zeros
    GaussianOperands o;
    load_material(a, g, o);
    const float m[3] = {a.means3D[3 * (size_t)g], a.means3D[3 * (size_t)g + 1], a.means3D[3 * (size_t)g + 2]};
    const float* Trow = a.shadows + (size_t)g * R;
    float dbase[3] = {0.f, 0.f, 0.f}, drough = 0.f, dmean[3] = {0.f, 0.f, 0.f};
    for (int v = 0; v < a.V; ++v) {
        const size_t row = (size_t)v * a.P + g;
        view_operands(o.n, a.viewdirs + 3 * row, o.V, o.vnorm, o.Ns);
        float gp[3], gs[3], gd[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            gp[c] = valid ? a.dL_dpbr[3 * row + c] : 0.f;
            gs[c] = valid && a.dL_dspecular ? a.dL_dspecular[3 * row + c] : 0.f;
            gd[c] = valid && a.dL_ddiffuse_light ? a.dL_ddiffuse_light[3 * row + c] : 0.f;
        }
        float dbase_v[3] = {0.f, 0.f, 0.f}, drough_v = 0.f, dmean_v[3] = {0.f, 0.f, 0.f}, dV[3] = {0.f, 0.f, 0.f};
        int col = 0;
        for (int j = 0; j < a.K; ++j) {
            const bool rect = (rect_mask >> j) & 1;
            const int n = rect ? a.M * a.M : 1;
            const uint32_t h = rect_hash(a.seed, (uint32_t)g, (uint32_t)j);
            const float* dir = s.dir + 3 * j;
            float acc[SL_SLOTS];
#pragma unroll
            for (int k = 0; k < SL_SLOTS; ++k) acc[k] = 0.f;
            for (int q = 0; q < n; ++q, ++col) {
                ShapedTerm t;
                shaped_term(rect, s, j, a.M, h, q, o, m, t);
                const float T = Trow[col];
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
                // GGX: roughness, view and the normalised direction it forms from l
                float dLn[3], dl[3];
                ggx_backward<true>(o.V, o.Ns, o, e, dfs, drough_v, dV, dLn);
                LightDir ll;
                ll.l[0] = t.d.l[0]; ll.l[1] = t.d.l[1]; ll.l[2] = t.d.l[2];
                ll.rn = sqrtf(ll.l[0] * ll.l[0] + ll.l[1] * ll.l[1] + ll.l[2] * ll.l[2]);
                const float lden = fmaxf(ll.rn, LIGHT_EPS);
#pragma unroll
                for (int c = 0; c < 3; ++c) ll.l[c] = ll.l[c] / lden;
                normalize_backward(ll, dLn, dl);
                const float dn = t.ndr >= 0.f ? dndi : 0.f;                   // clamp(min=0) passes the gradient at 0
#pragma unroll
                for (int c = 0; c < 3; ++c) dl[c] += dn * o.n[c];
                // the weight: E = color * wgt
                float dr2 = -dwgt * t.wgt / t.r2c;
                if (rect) {
                    const float k = (float)(a.M * a.M) * t.r2c;
                    const float ce = fmaxf(t.ce_r, 0.f);
                    acc[15] += dwgt * ce / k;                                  // dL/dA
                    const float dce = t.ce_r >= 0.f ? dwgt * s.sc[j] / k : 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) { acc[12 + c] -= dce * t.d.l[c]; dl[c] -= dce * dir[c]; }
                } else {
                    const float dx = dwgt / t.r2c * 6.0f * t.x * (1.0f - t.x);
                    const float dxr = (t.xr >= 0.f && t.xr <= 1.f) ? dx : 0.f;
                    const float dnum = dxr / s.sc[j];
                    const float dden = s.live[j] != 0.f ? -dxr * t.xr / s.sc[j] : 0.f;
                    acc[6] += dden; acc[7] -= dden + dnum;                    // cos_inner, cos_outer
#pragma unroll
                    for (int c = 0; c < 3; ++c) { acc[3 + c] -= dnum * t.d.l[c]; dl[c] -= dnum * dir[c]; }
                }
                if (!(t.d.r2 >= LIGHT_R2_MIN)) dr2 = 0.f;
                float dw[3];
                normalize_backward(t.d, dl, dw);
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float dy = dw[c] + 2.0f * t.d.w[c] * dr2;
                    dmean_v[c] -= dy;
                    acc[c] += dy;
                    if (rect) { acc[3 + c] += t.st[0] * dy; acc[6 + c] += t.st[1] * dy; }
                }
            }
            // the light's gradient: summed over the warp (fixed butterfly), added to the warp's row by lane 0
#pragma unroll
            for (int k = 0; k < SL_SLOTS; ++k) {
                const float x = warp_sum(valid ? acc[k] : 0.f);
                if (lane == 0) sAcc[warp][SL_SLOTS * j + k] += x;
            }
        }
        if (valid) {
            const float vd = o.V[0] * dV[0] + o.V[1] * dV[1] + o.V[2] * dV[2];
#pragma unroll
            for (int c = 0; c < 3; ++c) a.dL_dviewdirs[3 * row + c] = (dV[c] - o.V[c] * vd) / o.vnorm;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) { dbase[c] += dbase_v[c]; dmean[c] += dmean_v[c]; }
        drough += drough_v;
    }
    if (valid) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { a.dL_dbase_color[3 * (size_t)g + c] = dbase[c]; a.dL_dmeans3D[3 * (size_t)g + c] = dmean[c]; }
        a.dL_droughness[g] = drough;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < SL_SLOTS * a.K; i += LS_THREADS) {
        float x = sAcc[0][i];
#pragma unroll
        for (int w = 1; w < LS_WARPS; ++w) x += sAcc[w][i];
        partial[(size_t)blockIdx.x * SL_SLOTS * a.K + i] = x;
    }
}

// One CTA per light: warp k sums slot k over the CTA partials in block order (lane-strided, then a fixed butterfly),
// then one thread applies the light-level chain rule and writes the light's gradients
__global__ void __launch_bounds__(32 * SL_SLOTS) shaped_reduce_kernel(const r3dg_shaped_light_args a, const uint32_t rect_mask,
                                                                      int blocks, const float* __restrict__ partial) {
    __shared__ float r[SL_SLOTS];
    const int j = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float x = 0.f;
    for (int b = lane; b < blocks; b += 32) x += partial[(size_t)b * SL_SLOTS * a.K + SL_SLOTS * j + k];
    x = warp_sum(x);
    if (lane == 0) r[k] = x;
    __syncthreads();
    if (threadIdx.x != 0) return;
    float da[3], db[3] = {0.f, 0.f, 0.f}, dcone[2] = {0.f, 0.f};
    const float u[3] = {a.a[3 * j], a.a[3 * j + 1], a.a[3 * j + 2]};
    if ((rect_mask >> j) & 1) {
        const float v[3] = {a.b[3 * j], a.b[3 * j + 1], a.b[3 * j + 2]};
        const float c[3] = {u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]};
        const float cn = sqrtf(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
        float dc[3];
        normalize3_backward(c, r + 12, dc);                               // n_e = normalize(u x v)
#pragma unroll
        for (int q = 0; q < 3; ++q) dc[q] += cn > 0.f ? r[15] * 4.0f * c[q] / cn : 0.f;   // A = 4 |u x v|
        // c = u x v:  dL/du = v x dc,  dL/dv = dc x u
        da[0] = r[3] + (v[1] * dc[2] - v[2] * dc[1]); da[1] = r[4] + (v[2] * dc[0] - v[0] * dc[2]); da[2] = r[5] + (v[0] * dc[1] - v[1] * dc[0]);
        db[0] = r[6] + (dc[1] * u[2] - dc[2] * u[1]); db[1] = r[7] + (dc[2] * u[0] - dc[0] * u[2]); db[2] = r[8] + (dc[0] * u[1] - dc[1] * u[0]);
    } else {
        normalize3_backward(u, r + 3, da);                                // a^ = normalize(axis)
        dcone[0] = r[6]; dcone[1] = r[7];
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        a.dL_dpos[3 * j + q] = r[q]; a.dL_da[3 * j + q] = da[q]; a.dL_db[3 * j + q] = db[q]; a.dL_dcolor[3 * j + q] = r[9 + q];
    }
    a.dL_dcone[2 * j] = dcone[0]; a.dL_dcone[2 * j + 1] = dcone[1];
}

// ---- shaped-light host launchers --------------------------------------------------------------
int launch_shaped_reduce(const r3dg_shaped_light_args& a, uint32_t rect_mask, int blocks, const float* partial,
                         cudaStream_t stream) {
    shaped_reduce_kernel<<<a.K, 32 * SL_SLOTS, 0, stream>>>(a, rect_mask, blocks, partial);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

size_t shade_shaped_lights_work_bytes(int P, int K) {
    return P <= 0 || K <= 0 ? 0 : (size_t)lights_blocks(P) * SL_SLOTS * K * sizeof(float);
}

// R of a valid argument record, -1 otherwise
static int shaped_args_rays(const r3dg_shaped_light_args* a) {
    if (!a || a->P < 0 || a->V < 1 || a->V > R3DG_MAX_VIEWS) return -1;
    const int R = shaped_rays(a->K, a->kind, a->M);
    if (R < 0) return -1;
    if (a->K > 0) {
        const uint32_t rm = rect_mask(a->K, a->kind), spots = ((a->K == 32 ? 0u : 1u << a->K) - 1u) & ~rm;
        if (!a->pos || !a->a || !a->color || (rm && !a->b) || (spots && !a->cone)) return -1;
    }
    if (a->P > 0 && (!a->means3D || !a->base_color || !a->roughness || !a->normals || !a->viewdirs || (a->K > 0 && !a->shadows)))
        return -1;
    return R;
}

int launch_shade_shaped_lights_forward(const r3dg_shaped_light_args* a, cudaStream_t stream, bool* launched) {
    *launched = false;
    const int R = shaped_args_rays(a);
    if (R < 0) return R3DG_ERR_BAD_ARG;
    if (a->P > 0 && (!a->pbr || !a->diffuse_light || !a->specular)) return R3DG_ERR_BAD_ARG;
    if (a->P == 0) return 0;
    if (a->K == 0) {
        const size_t n = (size_t)a->V * a->P * 3 * sizeof(float);
        R3DG_CUDA_TRY(cudaMemsetAsync(a->pbr, 0, n, stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->diffuse_light, 0, n, stream));
        R3DG_CUDA_TRY(cudaMemsetAsync(a->specular, 0, n, stream));
        return 0;
    }
    shaped_fwd_kernel<<<lights_blocks(a->P), LS_THREADS, 0, stream>>>(*a, rect_mask(a->K, a->kind), R);
    R3DG_CUDA_TRY(cudaGetLastError());
    *launched = true;
    return 0;
}

int launch_shade_shaped_lights_backward(const r3dg_shaped_light_args* a, cudaStream_t stream, bool* launched) {
    *launched = false;
    const int R = shaped_args_rays(a);
    if (R < 0) return R3DG_ERR_BAD_ARG;
    if (a->P > 0 && (!a->dL_dpbr || !a->dL_dbase_color || !a->dL_droughness || !a->dL_dviewdirs || !a->dL_dmeans3D))
        return R3DG_ERR_BAD_ARG;
    if (a->K > 0 && (!a->dL_dpos || !a->dL_da || !a->dL_db || !a->dL_dcolor || !a->dL_dcone)) return R3DG_ERR_BAD_ARG;
    const size_t need = shade_shaped_lights_work_bytes(a->P, a->K);
    if (need > 0 && (!a->work || a->work_bytes < need)) return R3DG_ERR_BAD_ARG;
    if (a->P == 0 || a->K == 0) {
        if (a->P > 0) {
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dbase_color, 0, (size_t)a->P * 3 * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_droughness, 0, (size_t)a->P * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dviewdirs, 0, (size_t)a->V * a->P * 3 * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dmeans3D, 0, (size_t)a->P * 3 * sizeof(float), stream));
        }
        if (a->K > 0) {
            const size_t n3 = (size_t)a->K * 3 * sizeof(float);
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dpos, 0, n3, stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_da, 0, n3, stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_db, 0, n3, stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dcolor, 0, n3, stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dcone, 0, (size_t)a->K * 2 * sizeof(float), stream));
        }
        return 0;
    }
    const int blocks = lights_blocks(a->P);
    const uint32_t rm = rect_mask(a->K, a->kind);
    float* partial = (float*)a->work;
    shaped_bwd_kernel<<<blocks, LS_THREADS, 0, stream>>>(*a, rm, R, partial);
    R3DG_CUDA_TRY(cudaGetLastError());
    const int rc = launch_shaped_reduce(*a, rm, blocks, partial, stream);
    if (rc != 0) return rc;
    *launched = true;
    return 0;
}

}  // namespace r3dg
