// Stage 3a of the hot path: the BRDF shading step `rendering_equation` (reference
// gaussian_renderer/neilf.py:339-371) with `GGX_specular` (:374-406), the lat-long environment
// lookup (scene/direct_light_map.py:70-83, scene/envmap.py:35-53) and `eval_sh` (utils/sh_utils.py
// :71-128) — ~40 elementwise PyTorch kernels over [P,N,3] tensors in the reference, whose autograd
// graph keeps >= 15 such tensors alive (SURVEY.md §3.4) — as ONE forward and ONE backward kernel.
//
// Design notes
//  * a group of 8 lanes per Gaussian (4 Gaussians per warp), lanes stride the N incident samples:
//    the baked [P,N,*] tensors (direction 12 B + visibility 4 B + area 4 B per sample — the only
//    per-sample HBM traffic) are read once per direction, rows of neighbouring Gaussians are
//    contiguous so the warp's loads stay coalesced; nothing of size [P,N,*] is written unless the
//    caller asks for the eval-only per-sample lights.  (One warp per Gaussian left 1-2 samples per
//    lane at the training sample counts N = 32 / 64 and paid 290 shuffles per Gaussian.)
//  * per-Gaussian operands (material, normal, view direction, 48 SH coefficients) live in
//    registers; the backward reduces its 48 SH-coefficient gradients with a transposed butterfly
//    (42 shuffles per 4 Gaussians) and the group writes the 192 B row contiguously;
//  * the (small) environment texture lives in shared memory of a persistent CTA; its gradient —
//    grid_sample's scatter-add of P*N*4 taps — is accumulated in warp-private shared-memory copies
//    without atomics (shading_eval.cuh, "environment-map gradient"), summed and flushed once per CTA;
//  * the backward recomputes the forward per sample instead of saving [P,N,*] activations.
#include <cstring>
#include "shading_eval.cuh"

namespace r3dg {

template <bool INC_REGS>
__device__ __forceinline__ void load_operands(const ShadeArgs& a, int g, GaussianOperands& o) {
    load_material(a, g, o);
    view_operands(o.n, a.viewdirs + 3 * (size_t)g, o.V, o.vnorm, o.Ns);
    if (INC_REGS) {
        const float4* ip = reinterpret_cast<const float4*>(a.incidents + 48 * (size_t)g);
#pragma unroll
        for (int q = 0; q < 12; ++q) { const float4 v = ip[q]; o.inc[4 * q] = v.x; o.inc[4 * q + 1] = v.y; o.inc[4 * q + 2] = v.z; o.inc[4 * q + 3] = v.w; }
    }
}

// Kernel variants (r3dg_tune "shade_fwd_variant" / "shade_bwd_variant"): where the per-Gaussian SH
// state lives.  0: registers.  1: the 48 incident-light coefficients of each group in shared memory
// (broadcast LDS.128 reads, -48 registers).  2 (backward): additionally the 48 per-lane gradient
// accumulators in shared memory ([48][threads], conflict-free), loaded back once per Gaussian for
// the group reduction.  Fewer registers = more resident warps for a kernel that is bound by the
// latency of its dependent arithmetic (acos / atan2 / divisions), not by HBM.

template <int G>
__device__ __forceinline__ void stage_incidents(const ShadeArgs& a, int g, float* slot, int sub) {
    const float4* src = reinterpret_cast<const float4*>(a.incidents + 48 * (size_t)g);
    float4* dst = reinterpret_cast<float4*>(slot);
    for (int q = sub; q < 12; q += G) dst[q] = src[q];
    __syncwarp();
}

template <bool SMEM_ENV, bool INC_SMEM, bool FAST, bool FILT>
__device__ __forceinline__ void eval_sample(const ShadeArgs& a, const EnvLevels& lv, const GaussianOperands& o, const float* __restrict__ env,
                                            const float* __restrict__ sinc, float dx, float dy, float dz, float vis, float omega,
                                            SampleEvalT<FILT>& e) {
    eval_env_any<SMEM_ENV>(a.transform, env, a, lv, omega, dx, dy, dz, vis, e);
    eval_local<INC_SMEM>(o, sinc, dx, dy, dz, e);
    eval_ggx<FAST>(o.V, o.Ns, o, dx, dy, dz, e);
}

template <bool SMEM_ENV, int G, int VAR, bool FILT>
__global__ void __launch_bounds__(SHADE_THREADS, VAR == 1 ? (FILT ? 5 : 6) : 1) shade_fwd_kernel(const ShadeArgs a, const EnvLevels lv) {
    extern __shared__ __align__(16) float s_fwd[];     // [incident slots (VAR 1)][env texture (SMEM_ENV)]
    constexpr int GPW = 32 / G;                    // Gaussians per warp
    constexpr int INC_FLOATS = VAR >= 1 ? SHADE_WARPS * GPW * SHADE_INC_STRIDE : 0;
    float* s_env = s_fwd + INC_FLOATS;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & (G - 1), grp = lane / G;
    float* sinc = s_fwd + (warp * GPW + grp) * SHADE_INC_STRIDE;
    if (SMEM_ENV) {
        for (int i = threadIdx.x; i < (FILT ? lv.total : a.He * a.We) * 3; i += SHADE_THREADS) s_env[i] = a.env[i];
        __syncthreads();
    }
    const float* env = SMEM_ENV ? s_env : a.env;
    const float invN = 1.0f / (float)a.N;
    const int units = (a.P + GPW - 1) / GPW;
    for (int u = blockIdx.x * SHADE_WARPS + warp; u < units; u += gridDim.x * SHADE_WARPS) {
        const int g_raw = u * GPW + grp;
        const bool valid = g_raw < a.P;
        const int g = valid ? g_raw : a.P - 1;      // idle groups of the last warp shade a copy, write nothing
        GaussianOperands o;
        load_operands<VAR == 0>(a, g, o);
        if (VAR >= 1) stage_incidents<G>(a, g, sinc, sub);
        float pbr[3] = {0, 0, 0}, spec[3] = {0, 0, 0}, diff[3] = {0, 0, 0}, ml[3] = {0, 0, 0}, mloc[3] = {0, 0, 0}, mg[3] = {0, 0, 0}, mv = 0;
        const size_t row = (size_t)g * a.N;
        for (int i = sub; i < a.N; i += G) {
            const float dx = a.dirs[3 * (row + i)], dy = a.dirs[3 * (row + i) + 1], dz = a.dirs[3 * (row + i) + 2];
            const float vis = a.visibility[row + i], area = a.areas[row + i];
            SampleEvalT<FILT> e;
            eval_sample<SMEM_ENV, (VAR >= 1), false>(a, lv, o, env, sinc, dx, dy, dz, vis, area * invN, e);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float loc = fmaxf(e.local_raw[c], 0.f);
                const float Lc = loc + e.glob[c];
                const float T = Lc * area * e.ndi;
                const float fd = o.base[c] / PI_F;
                pbr[c] += (fd + e.fs) * T; spec[c] += e.fs * T; diff[c] += T;
                ml[c] += Lc; mloc[c] += loc; mg[c] += e.glob[c];
                if (a.s_lights && valid) { a.s_lights[3 * (row + i) + c] = Lc; a.s_local[3 * (row + i) + c] = loc; a.s_global[3 * (row + i) + c] = e.glob[c]; }
            }
            mv += vis;
        }
        __syncwarp();
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            pbr[c] = group_sum<G>(pbr[c]); spec[c] = group_sum<G>(spec[c]); diff[c] = group_sum<G>(diff[c]);
            if (a.mean_lights) { ml[c] = group_sum<G>(ml[c]); mloc[c] = group_sum<G>(mloc[c]); mg[c] = group_sum<G>(mg[c]); }
        }
        if (a.mean_vis) mv = group_sum<G>(mv);
        if (sub == 0 && valid) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                a.pbr[3 * (size_t)g + c] = pbr[c] * invN; a.specular[3 * (size_t)g + c] = spec[c] * invN; a.diffuse[3 * (size_t)g + c] = diff[c] * invN;
                if (a.mean_lights) { a.mean_lights[3 * (size_t)g + c] = ml[c] * invN; a.mean_local[3 * (size_t)g + c] = mloc[c] * invN; a.mean_global[3 * (size_t)g + c] = mg[c] * invN; }
            }
            if (a.mean_vis) a.mean_vis[g] = mv * invN;
        }
    }
}

// resident CTAs the register allocation is pinned to: variant 1 -> 3 (<= 168 registers); variant 2 ->
// 3 with the warp-private env copies (67 KB of shared memory per CTA) or the deterministic modes (their fixed-point
// conversion spills at 102 registers), 5 otherwise (<= 102 registers; 4 in the filtered mode, whose 8 env taps spill
// at 102)
template <int ENV_MODE, int G, int VAR, bool FILT>
__global__ void __launch_bounds__(SHADE_THREADS, VAR == 0 ? 1 : VAR == 1 ? 3 : (ENV_MODE <= 1 ? (FILT ? 4 : 5) : 3))
shade_bwd_kernel(const ShadeArgs a, const EnvLevels lv) {
    extern __shared__ __align__(16) float s_bwd[];    // [incident slots (VAR >= 1)][gradient accumulators (VAR 2)][env ...]
    constexpr bool SMEM_ENV = EnvGrad<ENV_MODE>::SMEM_ENV;
    constexpr int GPW = 32 / G;
    constexpr int INC_FLOATS = VAR >= 1 ? SHADE_WARPS * GPW * SHADE_INC_STRIDE : 0;
    constexpr int DINC_FLOATS = VAR == 2 ? 48 * SHADE_THREADS : 0;
    float* s_mem = s_bwd + INC_FLOATS + DINC_FLOATS;
    float* sinc = s_bwd + ((threadIdx.x >> 5) * GPW + (threadIdx.x & 31) / G) * SHADE_INC_STRIDE;
    float4* acc4 = reinterpret_cast<float4*>(s_bwd + INC_FLOATS) + threadIdx.x;    // VAR 2
    constexpr int VP = (48 + G - 1) / G * G;         // SH-gradient row padded to a multiple of G
    constexpr int RQ = VP / G;                       // finished components per lane
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & (G - 1), grp = lane / G;
    EnvGrad<ENV_MODE> eg(a, s_mem, warp, FILT ? lv.total : a.He * a.We);
    const float invN = 1.0f / (float)a.N;
    const int units = (a.P + GPW - 1) / GPW;
    for (int u = blockIdx.x * SHADE_WARPS + warp; u < units; u += gridDim.x * SHADE_WARPS) {
        const int g_raw = u * GPW + grp;
        const bool valid = g_raw < a.P;
        const int g = valid ? g_raw : a.P - 1;
        GaussianOperands o;
        load_operands<VAR == 0>(a, g, o);
        if (VAR >= 1) stage_incidents<G>(a, g, sinc, sub);
        float gp[3], gs[3], gd[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            gp[c] = a.g_pbr[3 * (size_t)g + c] * invN;
            gs[c] = a.g_specular ? a.g_specular[3 * (size_t)g + c] * invN : 0.f;
            gd[c] = a.g_diffuse ? a.g_diffuse[3 * (size_t)g + c] * invN : 0.f;
        }
        float dbase[3] = {0, 0, 0}, drough = 0.f, dV[3] = {0, 0, 0};
        float dinc[VP];
#pragma unroll
        for (int q = 0; q < VP; ++q) dinc[q] = 0.f;
        if (VAR == 2) {
#pragma unroll
            for (int q = 0; q < 12; ++q) acc4[q * SHADE_THREADS] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        const size_t row = (size_t)g * a.N;
        for (int i0 = 0; i0 < a.N; i0 += G) {          // warp-uniform trip count (collectives inside in ENV_TAG mode)
            const bool act = valid && (i0 + sub) < a.N;
            const int i = (i0 + sub) < a.N ? (i0 + sub) : a.N - 1;
            const float dx = a.dirs[3 * (row + i)], dy = a.dirs[3 * (row + i) + 1], dz = a.dirs[3 * (row + i) + 2];
            const float vis = a.visibility[row + i], area = a.areas[row + i];
            SampleEvalT<FILT> e;
            eval_sample<SMEM_ENV, (VAR >= 1), true>(a, lv, o, eg.env, sinc, dx, dy, dz, vis, area * invN, e);
            float dfs = 0.f;
            float dG[3], dLg[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float loc = fmaxf(e.local_raw[c], 0.f);
                const float T = (loc + e.glob[c]) * area * e.ndi;
                const float fd = o.base[c] * INV_PI_F;
                const float dT = act ? gp[c] * (fd + e.fs) + gs[c] * e.fs + gd[c] : 0.f;
                if (act) { dbase[c] += gp[c] * T * INV_PI_F; dfs += (gp[c] + gs[c]) * T; }
                const float dL = dT * area * e.ndi;
                dLg[c] = (act && e.local_raw[c] >= 0.f) ? dL : 0.f;  // clamp_min(0) passes the gradient at equality
                if (VAR != 2 && dLg[c] != 0.f) {
#pragma unroll
                    for (int k = 0; k < 16; ++k) dinc[3 * k + c] = fmaf(dL, e.w[k], dinc[3 * k + c]);
                }
                dG[c] = act ? dL * vis : 0.f;                        // -> env texels (grid_sample backward)
            }
            if (VAR == 2) accumulate_dinc(acc4, dLg, e.w);
            eg.scatter(a, e.taps, dG, lane);
            if (act) ggx_backward(o.V, o.Ns, o, e, dfs, drough, dV);
        }
        __syncwarp();
        // ---- group reduction and per-Gaussian outputs ---------------------------------------------
#pragma unroll
        for (int c = 0; c < 3; ++c) { dbase[c] = group_sum<G>(dbase[c]); dV[c] = group_sum<G>(dV[c]); }
        drough = group_sum<G>(drough);
        if (VAR == 2) {
#pragma unroll
            for (int q = 0; q < 12; ++q) { const float4 v = acc4[q * SHADE_THREADS]; dinc[4 * q] = v.x; dinc[4 * q + 1] = v.y; dinc[4 * q + 2] = v.z; dinc[4 * q + 3] = v.w; }
        }
        group_reduce_scatter<G, VP>(dinc, sub);        // lane `sub` now owns components [sub*RQ, sub*RQ + RQ)
        if (valid) {
            if (sub == 0) {
                const float vd = o.V[0] * dV[0] + o.V[1] * dV[1] + o.V[2] * dV[2];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    a.d_base[3 * (size_t)g + c] = dbase[c];
                    a.d_view[3 * (size_t)g + c] = (dV[c] - o.V[c] * vd) / o.vnorm;        // through V = normalize(viewdirs)
                }
                a.d_rough[g] = drough;
            }
            float* dp = a.d_incidents + 48 * (size_t)g + sub * RQ;    // the group writes the 192 B row contiguously
            if (RQ % 2 == 0) {
#pragma unroll
                for (int q = 0; q < RQ; q += 2)
                    if (sub * RQ + q < 48) *reinterpret_cast<float2*>(dp + q) = make_float2(dinc[q], dinc[q + 1]);
            } else {
#pragma unroll
                for (int q = 0; q < RQ; ++q)
                    if (sub * RQ + q < 48) dp[q] = dinc[q];
            }
        }
    }
    eg.flush(a);
}

// deterministic mode: the largest |cotangent| of the call over dL_dpbr, dL_ddiffuse_light and dL_dspecular (n floats
// each, NULL skipped) as float bits into *scale (zeroed), by atomicMax: exact and order-independent
__global__ void __launch_bounds__(256) det_scale_kernel(size_t n, const float* __restrict__ g0, const float* __restrict__ g1,
                                                        const float* __restrict__ g2, uint32_t* __restrict__ scale) {
    uint32_t m = 0u;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        m = max(m, det_abs_bits(g0[i]));
        if (g1) m = max(m, det_abs_bits(g1[i]));
        if (g2) m = max(m, det_abs_bits(g2[i]));
    }
    det_max_bits(scale, m);
}

// deterministic mode: dL/denv from its accumulators, every element written
__global__ void __launch_bounds__(256) det_env_kernel(const DetAcc acc, const uint32_t* __restrict__ scale, float* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < acc.n) out[i] = det_load(acc, i, det_scale_exp(*scale));
}

void launch_det_scale(const ShadeArgs& a, size_t n, int num_sms, cudaStream_t stream) {
    const unsigned blocks = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)4 * num_sms);
    det_scale_kernel<<<blocks, 256, 0, stream>>>(n, a.g_pbr, a.g_diffuse, a.g_specular, a.det_scale);
}

int launch_det_env(const ShadeArgs& a, cudaStream_t stream) {
    det_env_kernel<<<(unsigned)((a.det.n + 255) / 256), 256, 0, stream>>>(a.det, a.det_scale, a.d_env);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

// ---- several views per call ----------------------------------------------------------------------
// V view directions of the same Gaussians and baked samples.  Per group and sample the view-independent part runs once
// (baked loads, env taps and global light, SH basis and local light, n.w, and T = L area n.w); a loop over the views
// of the launch then runs GGX_specular forward (and backward).  One configuration: the default one-view one (groups of
// 8 lanes, incident SH coefficients staged in shared memory, the backward's 48 SH-gradient accumulators in shared
// memory).  A launch takes at most SHADE_VIEW_CHUNK views; each group keeps the operands of those views in a slot of
// shared memory, and each lane its per-view partial sums.  The forward runs each view's arithmetic in the one-view
// kernel's order, so every view's outputs equal a one-view call's bit for bit.
#define SHADE_VIEW_CHUNK 8
#define VIEW_FWD_SLOT 8           // floats per view and group: V[3], Ns[3] (padded)
#define VIEW_BWD_SLOT 16          // V[3], Ns[3], dL/dpbr, dL/dspecular, dL/ddiffuse_light (each [3], times 1/N), |viewdir|

struct ViewChunk {
    int v0, nv;                   // first view of the launch and its view count (<= SHADE_VIEW_CHUNK)
    int per_view_transform;       // forward: the env transform holds one [3,3] per view
    int accumulate;               // backward: add the leaf gradients to the earlier launches' (0: write them)
};

// per-lane partial sums of one view in the forward: pbr, specular, diffuse (+ mean lights, mean global with per-view transforms)
__host__ __device__ inline int view_fwd_sums(bool per_view_means) { return per_view_means ? 15 : 9; }

template <bool SMEM_ENV, bool FILT>
__global__ void __launch_bounds__(SHADE_THREADS, 3) shade_views_fwd_kernel(const ShadeArgs a, const ViewChunk vc, const EnvLevels lv) {
    constexpr int G = 8, GPW = 32 / G;
    constexpr int INC_FLOATS = SHADE_WARPS * GPW * SHADE_INC_STRIDE;
    constexpr int SLOT_FLOATS = SHADE_WARPS * GPW * SHADE_VIEW_CHUNK * VIEW_FWD_SLOT;
    extern __shared__ __align__(16) float s_vfwd[];   // [incident slots][view slots][per-lane sums K][view][threads][env]
    const bool pvt = vc.per_view_transform != 0, means = a.mean_lights != nullptr;
    const int K = view_fwd_sums(pvt && means);
    float* s_acc = s_vfwd + INC_FLOATS + SLOT_FLOATS;
    float* s_env = s_acc + K * SHADE_VIEW_CHUNK * SHADE_THREADS;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & (G - 1), grp = lane / G;
    float* sinc = s_vfwd + (warp * GPW + grp) * SHADE_INC_STRIDE;
    float* slot = s_vfwd + INC_FLOATS + (warp * GPW + grp) * SHADE_VIEW_CHUNK * VIEW_FWD_SLOT;
    if (SMEM_ENV) {
        for (int i = threadIdx.x; i < (FILT ? lv.total : a.He * a.We) * 3; i += SHADE_THREADS) s_env[i] = a.env[i];
        __syncthreads();
    }
    const float* env = SMEM_ENV ? s_env : a.env;
    const float invN = 1.0f / (float)a.N;
    const int units = (a.P + GPW - 1) / GPW;
    for (int u = blockIdx.x * SHADE_WARPS + warp; u < units; u += gridDim.x * SHADE_WARPS) {
        const int g_raw = u * GPW + grp;
        const bool valid = g_raw < a.P;
        const int g = valid ? g_raw : a.P - 1;
        GaussianOperands o;
        load_material(a, g, o);
        stage_incidents<G>(a, g, sinc, sub);
        if (sub < vc.nv) {
            float* vs = slot + sub * VIEW_FWD_SLOT;
            float vnorm;
            view_operands(o.n, a.viewdirs + 3 * ((size_t)(vc.v0 + sub) * a.P + g), vs, vnorm, vs + 3);
        }
        for (int j = 0; j < K * vc.nv; ++j) s_acc[j * SHADE_THREADS + threadIdx.x] = 0.f;
        __syncwarp();
        float ml[3] = {0, 0, 0}, mloc[3] = {0, 0, 0}, mg[3] = {0, 0, 0}, mv = 0;
        const size_t row = (size_t)g * a.N;
        for (int i = sub; i < a.N; i += G) {
            const float dx = a.dirs[3 * (row + i)], dy = a.dirs[3 * (row + i) + 1], dz = a.dirs[3 * (row + i) + 2];
            const float vis = a.visibility[row + i], area = a.areas[row + i];
            SampleEvalT<FILT> e;
            if (!pvt) eval_env_any<SMEM_ENV>(a.transform, env, a, lv, area * invN, dx, dy, dz, vis, e);
            eval_local<true>(o, sinc, dx, dy, dz, e);
            float loc[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                loc[c] = fmaxf(e.local_raw[c], 0.f);
                mloc[c] += loc[c];
                if (!pvt) { ml[c] += loc[c] + e.glob[c]; mg[c] += e.glob[c]; }
            }
            mv += vis;
            for (int v = 0; v < vc.nv; ++v) {
                const float* vs = slot + v * VIEW_FWD_SLOT;
                if (pvt) eval_env_any<SMEM_ENV>(a.transform + 9 * (size_t)(vc.v0 + v), env, a, lv, area * invN, dx, dy, dz, vis, e);
                eval_ggx<false>(vs, vs + 3, o, dx, dy, dz, e);
                float* acc = s_acc + v * K * SHADE_THREADS + threadIdx.x;
#pragma unroll
                for (int c = 0; c < 3; ++c) {                 // the one-view kernel's expressions
                    const float Lc = loc[c] + e.glob[c];
                    const float T = Lc * area * e.ndi;
                    const float fd = o.base[c] / PI_F;
                    acc[c * SHADE_THREADS] += (fd + e.fs) * T; acc[(3 + c) * SHADE_THREADS] += e.fs * T; acc[(6 + c) * SHADE_THREADS] += T;
                    if (K == 15) { acc[(9 + c) * SHADE_THREADS] += Lc; acc[(12 + c) * SHADE_THREADS] += e.glob[c]; }
                }
            }
        }
        __syncwarp();
        if (means) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                mloc[c] = group_sum<G>(mloc[c]);
                if (!pvt) { ml[c] = group_sum<G>(ml[c]); mg[c] = group_sum<G>(mg[c]); }
            }
            mv = group_sum<G>(mv);
        }
        for (int v = 0; v < vc.nv; ++v) {
            const float* acc = s_acc + v * K * SHADE_THREADS + threadIdx.x;
            float r[15];
#pragma unroll
            for (int j = 0; j < 15; ++j) if (j < K) r[j] = group_sum<G>(acc[j * SHADE_THREADS]);
            if (sub == 0 && valid) {
                const size_t vg = (size_t)(vc.v0 + v) * a.P + g;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    a.pbr[3 * vg + c] = r[c] * invN; a.specular[3 * vg + c] = r[3 + c] * invN; a.diffuse[3 * vg + c] = r[6 + c] * invN;
                    if (means) {
                        a.mean_lights[3 * vg + c] = (pvt ? r[9 + c] : ml[c]) * invN; a.mean_local[3 * vg + c] = mloc[c] * invN;
                        a.mean_global[3 * vg + c] = (pvt ? r[12 + c] : mg[c]) * invN;
                    }
                }
                if (means) a.mean_vis[vg] = mv * invN;
            }
        }
    }
}

// Backward over the views of one launch, with the environment transform shared by all views.  Per sample the view
// loop sums dT = sum_v dL/dT_v; the SH-gradient contraction and the env scatter then run once on that sum, and dL/dbase
// uses the summed dL/dpbr.  dL/dviewdirs stays per view.  `accumulate` adds the leaf gradients to those of the earlier
// launches, in launch order (a fixed fold, so the deterministic mode stays reproducible).
template <int ENV_MODE, bool FILT>
__global__ void __launch_bounds__(SHADE_THREADS, 3) shade_views_bwd_kernel(const ShadeArgs a, const ViewChunk vc, const EnvLevels lv) {
    constexpr bool SMEM_ENV = EnvGrad<ENV_MODE>::SMEM_ENV;
    constexpr int G = 8, GPW = 32 / G, RQ = 48 / G;
    constexpr int INC_FLOATS = SHADE_WARPS * GPW * SHADE_INC_STRIDE;
    constexpr int DINC_FLOATS = 48 * SHADE_THREADS;
    constexpr int SLOT_FLOATS = SHADE_WARPS * GPW * SHADE_VIEW_CHUNK * VIEW_BWD_SLOT;
    constexpr int DV_FLOATS = 3 * SHADE_VIEW_CHUNK * SHADE_THREADS;
    // [incident slots][SH-gradient accumulators][view slots][per-lane dL/dV: 3][view][threads][env ...]
    extern __shared__ __align__(16) float s_vbwd[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & (G - 1), grp = lane / G;
    float* sinc = s_vbwd + (warp * GPW + grp) * SHADE_INC_STRIDE;
    float4* acc4 = reinterpret_cast<float4*>(s_vbwd + INC_FLOATS) + threadIdx.x;
    float* slot = s_vbwd + INC_FLOATS + DINC_FLOATS + (warp * GPW + grp) * SHADE_VIEW_CHUNK * VIEW_BWD_SLOT;
    float* s_dv = s_vbwd + INC_FLOATS + DINC_FLOATS + SLOT_FLOATS + threadIdx.x;
    EnvGrad<ENV_MODE> eg(a, s_vbwd + INC_FLOATS + DINC_FLOATS + SLOT_FLOATS + DV_FLOATS, warp, FILT ? lv.total : a.He * a.We);
    const float invN = 1.0f / (float)a.N;
    const int units = (a.P + GPW - 1) / GPW;
    for (int u = blockIdx.x * SHADE_WARPS + warp; u < units; u += gridDim.x * SHADE_WARPS) {
        const int g_raw = u * GPW + grp;
        const bool valid = g_raw < a.P;
        const int g = valid ? g_raw : a.P - 1;
        GaussianOperands o;
        load_material(a, g, o);
        stage_incidents<G>(a, g, sinc, sub);
        if (sub < vc.nv) {
            float* vs = slot + sub * VIEW_BWD_SLOT;
            const size_t vg = (size_t)(vc.v0 + sub) * a.P + g;
            view_operands(o.n, a.viewdirs + 3 * vg, vs, vs[15], vs + 3);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                vs[6 + c] = a.g_pbr[3 * vg + c] * invN;
                vs[9 + c] = a.g_specular ? a.g_specular[3 * vg + c] * invN : 0.f;
                vs[12 + c] = a.g_diffuse ? a.g_diffuse[3 * vg + c] * invN : 0.f;
            }
        }
#pragma unroll
        for (int q = 0; q < 12; ++q) acc4[q * SHADE_THREADS] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < 3 * vc.nv; ++j) s_dv[j * SHADE_THREADS] = 0.f;
        __syncwarp();
        float gp_sum[3] = {0, 0, 0};
        for (int v = 0; v < vc.nv; ++v)
#pragma unroll
            for (int c = 0; c < 3; ++c) gp_sum[c] += slot[v * VIEW_BWD_SLOT + 6 + c];
        float dbase[3] = {0, 0, 0}, drough = 0.f;
        const size_t row = (size_t)g * a.N;
        for (int i0 = 0; i0 < a.N; i0 += G) {          // warp-uniform trip count (collectives inside in ENV_TAG mode)
            const bool act = valid && (i0 + sub) < a.N;
            const int i = (i0 + sub) < a.N ? (i0 + sub) : a.N - 1;
            const float dx = a.dirs[3 * (row + i)], dy = a.dirs[3 * (row + i) + 1], dz = a.dirs[3 * (row + i) + 2];
            const float vis = a.visibility[row + i], area = a.areas[row + i];
            SampleEvalT<FILT> e;
            eval_env_any<SMEM_ENV>(a.transform, eg.env, a, lv, area * invN, dx, dy, dz, vis, e);
            eval_local<true>(o, sinc, dx, dy, dz, e);
            float T[3], dT[3] = {0, 0, 0};
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                T[c] = (fmaxf(e.local_raw[c], 0.f) + e.glob[c]) * area * e.ndi;
                if (act) dbase[c] += gp_sum[c] * T[c] * INV_PI_F;
            }
            if (act) {
                for (int v = 0; v < vc.nv; ++v) {
                    const float* vs = slot + v * VIEW_BWD_SLOT;
                    eval_ggx<true>(vs, vs + 3, o, dx, dy, dz, e);
                    float dfs = 0.f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float gp = vs[6 + c], gs = vs[9 + c];
                        dT[c] += gp * (o.base[c] * INV_PI_F + e.fs) + gs * e.fs + vs[12 + c];
                        dfs += (gp + gs) * T[c];
                    }
                    float dV[3] = {0, 0, 0};
                    ggx_backward(vs, vs + 3, o, e, dfs, drough, dV);
#pragma unroll
                    for (int c = 0; c < 3; ++c) s_dv[(3 * v + c) * SHADE_THREADS] += dV[c];
                }
            }
            float dG[3], dLg[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float dL = dT[c] * area * e.ndi;
                dLg[c] = (act && e.local_raw[c] >= 0.f) ? dL : 0.f;  // clamp_min(0) passes the gradient at equality
                dG[c] = act ? dL * vis : 0.f;                        // -> env texels (grid_sample backward)
            }
            accumulate_dinc(acc4, dLg, e.w);
            eg.scatter(a, e.taps, dG, lane);
        }
        __syncwarp();
        // ---- group reduction and per-Gaussian outputs ---------------------------------------------
#pragma unroll
        for (int c = 0; c < 3; ++c) dbase[c] = group_sum<G>(dbase[c]);
        drough = group_sum<G>(drough);
        for (int v = 0; v < vc.nv; ++v) {
            float dV[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) dV[c] = group_sum<G>(s_dv[(3 * v + c) * SHADE_THREADS]);
            if (sub == 0 && valid) {
                const float* vs = slot + v * VIEW_BWD_SLOT;
                const float vd = vs[0] * dV[0] + vs[1] * dV[1] + vs[2] * dV[2];
                float* dview = a.d_view + 3 * ((size_t)(vc.v0 + v) * a.P + g);
#pragma unroll
                for (int c = 0; c < 3; ++c) dview[c] = (dV[c] - vs[c] * vd) / vs[15];      // through V = normalize(viewdirs)
            }
        }
        float dinc[48];
#pragma unroll
        for (int q = 0; q < 12; ++q) { const float4 v = acc4[q * SHADE_THREADS]; dinc[4 * q] = v.x; dinc[4 * q + 1] = v.y; dinc[4 * q + 2] = v.z; dinc[4 * q + 3] = v.w; }
        group_reduce_scatter<G, 48>(dinc, sub);        // lane `sub` now owns components [sub*RQ, sub*RQ + RQ)
        if (valid) {
            if (sub == 0) {
#pragma unroll
                for (int c = 0; c < 3; ++c) a.d_base[3 * (size_t)g + c] = vc.accumulate ? a.d_base[3 * (size_t)g + c] + dbase[c] : dbase[c];
                a.d_rough[g] = vc.accumulate ? a.d_rough[g] + drough : drough;
            }
            float* dp = a.d_incidents + 48 * (size_t)g + sub * RQ;    // the group writes the 192 B row contiguously
#pragma unroll
            for (int q = 0; q < RQ; q += 2) {
                float2 w = make_float2(dinc[q], dinc[q + 1]);
                if (vc.accumulate) { const float2 p = *reinterpret_cast<const float2*>(dp + q); w.x = p.x + w.x; w.y = p.y + w.y; }
                *reinterpret_cast<float2*>(dp + q) = w;
            }
        }
    }
    eg.flush(a);
}

// ---- launch ---------------------------------------------------------------------------------------
// tuning knobs (A/B measurements and tests of the non-default paths), changed at run time through r3dg_tune
// (include/r3dg_b200.h); each starts at its default
struct ShadeKnob { const char* key; int lo, hi, value; };
static ShadeKnob g_knobs[] = {
    {"shade_group", 8, 32, 8},            // lanes per Gaussian: 8, 16 or 32
    // defaults = the fastest combination measured during development (tools/bench_stage3.py times the variants;
    // variant 2 with shared atomics fits more CTAs per SM than with tagged copies)
    {"shade_env_mode", 0, 2, ENV_CAS},    // highest env-gradient mode allowed
    {"shade_fwd_variant", 0, 1, 1},       // 1: incident SH coefficients in shared memory
    {"shade_bwd_variant", 0, 2, 2},       // 1: as forward; 2: + gradient accumulators in shared memory
};
static bool knob_ok(const ShadeKnob& k, int v) {
    if (v < k.lo || v > k.hi) return false;
    return strcmp(k.key, "shade_group") != 0 || v == 8 || v == 16 || v == 32;
}
static int knob(int i) { return g_knobs[i].value; }
int shade_tune(const char* key, int value, int* previous) {
    for (int i = 0; i < (int)(sizeof(g_knobs) / sizeof(g_knobs[0])); ++i) {
        if (strcmp(key, g_knobs[i].key)) continue;
        *previous = knob(i);
        if (!knob_ok(g_knobs[i], value)) return R3DG_ERR_BAD_ARG;
        g_knobs[i].value = value;
        return 0;
    }
    return R3DG_ERR_UNSUPPORTED;
}

template <bool SMEM, bool FILT>
static int launch_fwd(const ShadeArgs& a, const EnvLevels& lv, int num_sms, size_t env_smem, cudaStream_t stream) {
    const int G = knob(0);
    const int var = G == 8 ? knob(2) : 0;              // the shared-memory variants are built for the default group width
    const size_t smem = env_smem + inc_slot_bytes(G, var);
    const int units = (a.P + 32 / G - 1) / (32 / G);
    if (G == 8) return var ? shade_launch(shade_fwd_kernel<SMEM, 8, 1, FILT>, a, units, num_sms, smem, stream, lv)
                           : shade_launch(shade_fwd_kernel<SMEM, 8, 0, FILT>, a, units, num_sms, smem, stream, lv);
    if (G == 16) return shade_launch(shade_fwd_kernel<SMEM, 16, 0, FILT>, a, units, num_sms, smem, stream, lv);
    return shade_launch(shade_fwd_kernel<SMEM, 32, 0, FILT>, a, units, num_sms, smem, stream, lv);
}

int launch_shade_forward(ShadeArgs a, const EnvLevels& lv, bool filt, int num_sms, cudaStream_t stream) {
    if (a.P <= 0) return 0;
    const size_t env_bytes = env_texels(a, lv, filt) * 3 * sizeof(float);
    const bool smem = env_bytes <= 40 * 1024;
    a.env_in_smem = smem;
    if (filt) return smem ? launch_fwd<true, true>(a, lv, num_sms, env_bytes, stream) : launch_fwd<false, true>(a, lv, num_sms, 0, stream);
    return smem ? launch_fwd<true, false>(a, lv, num_sms, env_bytes, stream) : launch_fwd<false, false>(a, lv, num_sms, 0, stream);
}

template <int MODE, bool FILT>
static int launch_bwd(const ShadeArgs& a, const EnvLevels& lv, int num_sms, size_t env_smem, cudaStream_t stream) {
    const int G = knob(0);
    const int var = G == 8 ? knob(3) : 0;
    const size_t smem = env_smem + inc_slot_bytes(G, var) + (var == 2 ? (size_t)48 * SHADE_THREADS * sizeof(float) : 0);
    const int units = (a.P + 32 / G - 1) / (32 / G);
    if (G == 8) return var == 2 ? shade_launch(shade_bwd_kernel<MODE, 8, 2, FILT>, a, units, num_sms, smem, stream, lv)
                     : var == 1 ? shade_launch(shade_bwd_kernel<MODE, 8, 1, FILT>, a, units, num_sms, smem, stream, lv)
                                : shade_launch(shade_bwd_kernel<MODE, 8, 0, FILT>, a, units, num_sms, smem, stream, lv);
    if (G == 16) return shade_launch(shade_bwd_kernel<MODE, 16, 0, FILT>, a, units, num_sms, smem, stream, lv);
    return shade_launch(shade_bwd_kernel<MODE, 32, 0, FILT>, a, units, num_sms, smem, stream, lv);
}

int launch_shade_backward(ShadeArgs a, const EnvLevels& lv, bool filt, int num_sms, cudaStream_t stream) {
    return shade_backward(a, 1, knob(1), env_texels(a, lv, filt), num_sms, stream, [&](auto mode, const ShadeArgs& x, size_t env_smem) {
        constexpr int M = decltype(mode)::value;
        return filt ? launch_bwd<M, true>(x, lv, num_sms, env_smem, stream) : launch_bwd<M, false>(x, lv, num_sms, env_smem, stream);
    });
}

// ---- several views: one launch per SHADE_VIEW_CHUNK views ------------------------------------------
static size_t view_slot_bytes(int slot_floats) { return (size_t)SHADE_WARPS * 4 * SHADE_VIEW_CHUNK * slot_floats * sizeof(float); }

int launch_shade_views_forward(ShadeArgs a, const EnvLevels& lv, bool filt, int V, int per_view_transform, int num_sms,
                               cudaStream_t stream) {
    if (a.P <= 0) return 0;
    const size_t env_bytes = env_texels(a, lv, filt) * 3 * sizeof(float);
    const bool smem_env = env_bytes <= 40 * 1024;     // as the one-view forward
    a.env_in_smem = smem_env;
    const int K = view_fwd_sums(per_view_transform && a.mean_lights);
    const size_t smem = inc_slot_bytes(8, 1) + view_slot_bytes(VIEW_FWD_SLOT) + (size_t)K * SHADE_VIEW_CHUNK * SHADE_THREADS * sizeof(float) +
                        (smem_env ? env_bytes : 0);
    const int units = (a.P + 3) / 4;
    for (int v0 = 0; v0 < V; v0 += SHADE_VIEW_CHUNK) {
        const ViewChunk vc{v0, V - v0 < SHADE_VIEW_CHUNK ? V - v0 : SHADE_VIEW_CHUNK, per_view_transform, 0};
        const int rc = filt ? (smem_env ? shade_launch(shade_views_fwd_kernel<true, true>, a, units, num_sms, smem, stream, vc, lv)
                                        : shade_launch(shade_views_fwd_kernel<false, true>, a, units, num_sms, smem, stream, vc, lv))
                            : (smem_env ? shade_launch(shade_views_fwd_kernel<true, false>, a, units, num_sms, smem, stream, vc, lv)
                                        : shade_launch(shade_views_fwd_kernel<false, false>, a, units, num_sms, smem, stream, vc, lv));
        if (rc) return rc;
    }
    return 0;
}

// the env-gradient mode as the one-view backward picks it at its default highest mode (the view kernels have no knobs)
int launch_shade_views_backward(ShadeArgs a, const EnvLevels& lv, bool filt, int V, int num_sms, cudaStream_t stream) {
    return shade_backward(a, V, ENV_CAS, env_texels(a, lv, filt), num_sms, stream, [&](auto mode, const ShadeArgs& x, size_t env_smem) {
        constexpr int M = decltype(mode)::value;
        if constexpr (M == ENV_TAG) return (int)R3DG_ERR_UNSUPPORTED;     // above the cap: never selected
        else {
            const size_t smem = inc_slot_bytes(8, 2) + (size_t)48 * SHADE_THREADS * sizeof(float) + view_slot_bytes(VIEW_BWD_SLOT) +
                                (size_t)3 * SHADE_VIEW_CHUNK * SHADE_THREADS * sizeof(float) + env_smem;
            for (int v0 = 0; v0 < V; v0 += SHADE_VIEW_CHUNK) {
                const ViewChunk vc{v0, V - v0 < SHADE_VIEW_CHUNK ? V - v0 : SHADE_VIEW_CHUNK, 0, v0 > 0};
                const int rc = filt ? shade_launch(shade_views_bwd_kernel<M, true>, x, (x.P + 3) / 4, num_sms, smem, stream, vc, lv)
                                    : shade_launch(shade_views_bwd_kernel<M, false>, x, (x.P + 3) / 4, num_sms, smem, stream, vc, lv);
                if (rc) return rc;
            }
            return 0;
        }
    });
}

}  // namespace r3dg

// ---- C ABI --------------------------------------------------------------------------------------
using namespace r3dg;
extern "C" {

static int fill_args(const r3dg_shade_args* s, ShadeArgs& a) {
    if (!s || s->P < 0 || s->N <= 0 || s->env_h <= 0 || s->env_w <= 0) return R3DG_ERR_BAD_ARG;
    if (s->V < 0 || s->V > R3DG_MAX_VIEWS) return R3DG_ERR_BAD_ARG;
    if (s->sh_coeffs != 16) return R3DG_ERR_UNSUPPORTED;          // incidents are degree-3 SH ([P,16,3]) in the reference
    a.P = s->P; a.N = s->N; a.He = s->env_h; a.We = s->env_w; a.env_in_smem = 0;
    a.base_color = s->base_color; a.roughness = s->roughness; a.normals = s->normals; a.viewdirs = s->viewdirs;
    a.incidents = s->incidents; a.env = s->env; a.transform = s->env_transform;
    a.visibility = s->visibility; a.dirs = s->incident_dirs; a.areas = s->incident_areas;
    a.pbr = s->pbr; a.diffuse = s->diffuse_light; a.specular = s->specular;
    a.mean_lights = s->mean_incident_lights; a.mean_local = s->mean_local_lights; a.mean_global = s->mean_global_lights;
    a.mean_vis = s->mean_visibility;
    a.s_lights = s->incident_lights; a.s_local = s->local_incident_lights; a.s_global = s->global_incident_lights;
    a.g_pbr = s->dL_dpbr; a.g_diffuse = s->dL_ddiffuse_light; a.g_specular = s->dL_dspecular;
    a.d_base = s->dL_dbase_color; a.d_rough = s->dL_droughness; a.d_view = s->dL_dviewdirs; a.d_incidents = s->dL_dincidents;
    a.d_env = s->dL_denv;
    a.det = DetAcc{nullptr, nullptr, 0};
    a.det_scale = nullptr;
    return 0;
}

// the filtered mode runs when a pyramid is given and the env has a coarser level; otherwise the call is the plain one
static bool filtered(const r3dg_shade_args* s, const EnvLevels& lv) { return s->env_pyramid && lv.L > 1; }

int r3dg_render_equation_forward(const r3dg_shade_args* s, r3dg_stream_t stream) {
    ShadeArgs a;
    int rc = fill_args(s, a);
    if (rc) return rc;
    if (a.P > 0 && (!a.pbr || !a.diffuse || !a.specular)) return R3DG_ERR_BAD_ARG;
    if ((a.mean_lights != nullptr) != (a.mean_local != nullptr) || (a.mean_lights != nullptr) != (a.mean_global != nullptr)) return R3DG_ERR_BAD_ARG;
    if ((a.s_lights != nullptr) != (a.s_local != nullptr) || (a.s_lights != nullptr) != (a.s_global != nullptr)) return R3DG_ERR_BAD_ARG;
    const EnvLevels lv = env_levels(a.He, a.We);
    const bool filt = filtered(s, lv);
    if (filt) a.env = s->env_pyramid;
    if (s->V > 1) {
        if (a.s_lights) return R3DG_ERR_UNSUPPORTED;               // no per-sample [V,P,N,3] outputs
        if (a.mean_lights && !a.mean_vis) return R3DG_ERR_BAD_ARG;
        return launch_shade_views_forward(a, lv, filt, s->V, s->transform_per_view && a.transform, num_sms(), (cudaStream_t)stream);
    }
    return launch_shade_forward(a, lv, filt, num_sms(), (cudaStream_t)stream);
}

int r3dg_render_equation_backward(const r3dg_shade_args* s, r3dg_stream_t stream) {
    ShadeArgs a;
    int rc = fill_args(s, a);
    if (rc) return rc;
    if (!a.g_pbr || !a.d_base || !a.d_rough || !a.d_view || !a.d_incidents || !a.d_env) return R3DG_ERR_BAD_ARG;
    if (s->env_pyramid && !s->dL_denv_pyramid) return R3DG_ERR_BAD_ARG;
    if (s->V > 1 && s->transform_per_view && a.transform) return R3DG_ERR_UNSUPPORTED;    // forward only
    const EnvLevels lv = env_levels(a.He, a.We);
    const bool filt = filtered(s, lv);
    float* d_env = a.d_env;
    if (filt) { a.env = s->env_pyramid; a.d_env = s->dL_denv_pyramid; }      // the kernels' gradient: every level
    if (s->deterministic) {
        const size_t need = s->env_pyramid ? r3dg_shade_filtered_det_bytes(a.He, a.We) : r3dg_shade_det_bytes(a.He, a.We);
        if (!s->det_work || s->det_work_bytes < need) return R3DG_ERR_BAD_ARG;
        const size_t n = env_texels(a, lv, filt) * 3;
        a.det = det_acc(s->det_work, n);
        a.det_scale = (uint32_t*)((char*)s->det_work + det_bytes(n));
    }
    const cudaStream_t st = (cudaStream_t)stream;
    rc = s->V > 1 ? launch_shade_views_backward(a, lv, filt, s->V, num_sms(), st) : launch_shade_backward(a, lv, filt, num_sms(), st);
    if (rc || !filt) return rc;
    return launch_env_pyramid_adjoint(lv, a.d_env, d_env, st);               // dL/denv through the pyramid
}

// the accumulators and the call's scale word
size_t r3dg_shade_det_bytes(int env_h, int env_w) {
    return env_h > 0 && env_w > 0 ? det_bytes((size_t)env_h * env_w * 3) + 256 : 0;
}

size_t r3dg_shade_filtered_det_bytes(int env_h, int env_w) {
    return env_h > 0 && env_w > 0 ? det_bytes(r3dg_env_pyramid_floats(env_h, env_w)) + 256 : 0;
}

}  // extern "C"
