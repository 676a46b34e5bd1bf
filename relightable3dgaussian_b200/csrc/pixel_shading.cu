// Per-pixel (deferred) shading (include/r3dg_b200.h, PIXEL SHADING; DESIGN.md §4.29): the shading step of shading.cu
// at every valid pixel of rasterized material images instead of at every Gaussian, so a highlight or a shadow edge
// can vary inside one Gaussian's footprint.
//
// A pixel is a "Gaussian row" of the shading step: its base colour, roughness, raw normal and incident SH come from
// planar [C,H,W] images, its view direction is campos - point, its N samples are the sampler's directions around its
// unit normal (regenerated here from the normal and the canonical sample table, never read) with area 2 pi, and its
// visibility is the pixel trace's T [V,N,H,W].  The kernels are the per-Gaussian default configuration (groups of 8
// lanes striding the samples, incident SH staged in shared memory, the backward's SH-gradient accumulators in shared
// memory) with the same per-sample code (shading_eval.cuh, brdf.cuh) and the same sums in the same order, so every
// forward output equals the per-Gaussian kernel's on the pixel as a row, bit for bit.  A group of masked pixels does
// no sample work and writes zeros.
#include "bvh.cuh"
#include "importance.cuh"
#include "shading_eval.cuh"

namespace r3dg {

#define PIX_G 8                          // lanes per pixel: the per-Gaussian kernels' default group
#define PIX_GPW (32 / PIX_G)
#define PIX_AREA 6.283185307179586f      // the sampler's area, 2 pi

// The per-pixel part of a call; the ShadeArgs record holds the images (P = H W pixels per view).
struct PixelView {
    int V, per_view_transform;
    const float *points, *campos;        // [V,3,HW], [V,3]
    const uint8_t* mask;                 // [V,HW] or NULL
};

// shared-memory floats of the canonical sample table, rounded up to 16 bytes
__host__ __device__ inline int sample_table_floats(int N) { return (3 * N + 3) & ~3; }

// The operands of pixel vq = v HW + q: material, raw normal, view operands of campos_v - point, and the unit normal
// the samples are rotated to.
__device__ __forceinline__ void load_pixel(const ShadeArgs& a, const PixelView& pv, int v, size_t q, GaussianOperands& o,
                                           float3& nh) {
    const size_t HW = (size_t)a.P;
    float vd[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const size_t k = (3 * (size_t)v + c) * HW + q;
        o.base[c] = a.base_color[k];
        o.n[c] = a.normals[k];
        vd[c] = pv.campos[3 * v + c] - pv.points[k];
    }
    o.rough = a.roughness[(size_t)v * HW + q];
    roughness_operands(o);
    view_operands(o.n, vd, o.V, o.vnorm, o.Ns);
    nh = unit_normal(o.n[0], o.n[1], o.n[2]);
}

// the pixel's 48 incident-light coefficients ([V,48,HW] planes) into its group's slot, or zeros without incidents
__device__ __forceinline__ void stage_pixel_incidents(const ShadeArgs& a, int v, size_t q, float* slot, int sub) {
    const size_t HW = (size_t)a.P;
    for (int j = sub; j < 48; j += PIX_G) slot[j] = a.incidents ? a.incidents[(48 * (size_t)v + j) * HW + q] : 0.f;
    __syncwarp();
}

// the local light and n.d of one sample (the shading step's, or zero light without incidents)
template <class E>
__device__ __forceinline__ void pixel_local(const ShadeArgs& a, const GaussianOperands& o, const float* sinc, float3 d, E& e) {
    if (a.incidents) {
        eval_local<true>(o, sinc, d.x, d.y, d.z, e);
    } else {
        e.local_raw[0] = e.local_raw[1] = e.local_raw[2] = 0.f;
        e.ndi = fmaxf(o.n[0] * d.x + o.n[1] * d.y + o.n[2] * d.z, 0.f);     // eval_local's n.w
    }
}

__device__ __forceinline__ const float* view_transform(const ShadeArgs& a, const PixelView& pv, int v) {
    return a.transform && pv.per_view_transform ? a.transform + 9 * (size_t)v : a.transform;
}

// the importance sampler's GGX frame of pixel vq (read only with GGX samples)
__device__ __forceinline__ GgxFrame pixel_ggx_frame(const ShadeArgs& a, const PixelView& pv, const ImportanceSampler& smp, int v,
                                                    size_t q, const GaussianOperands& o, float3 nh) {
    GgxFrame f{};
    if (smp.n_ggx > 0) {
        const size_t HW = (size_t)a.P;
        f = ggx_frame(nh, sub_(pv.campos[3 * v], pv.points[3 * v * HW + q]), sub_(pv.campos[3 * v + 1], pv.points[(3 * v + 1) * HW + q]),
                      sub_(pv.campos[3 * v + 2], pv.points[(3 * v + 2) * HW + q]), o.rough);
    }
    return f;
}

// IS: the importance sampler's directions and areas (include/r3dg_b200.h, IMPORTANCE SAMPLING) instead of the canonical
// sample table's with area 2 pi; the same sums in the same order
template <bool SMEM_ENV, bool FILT, bool IS>
__global__ void __launch_bounds__(SHADE_THREADS, FILT ? 5 : 6) pixel_shade_fwd_kernel(const ShadeArgs a, const PixelView pv,
                                                                                      const EnvLevels lv, ImportanceSampler smp) {
    extern __shared__ __align__(16) float s_pfwd[];     // [incident slots][sample table][env texture (SMEM_ENV)]
    constexpr int INC_FLOATS = SHADE_WARPS * PIX_GPW * SHADE_INC_STRIDE;
    float3* s_smp = reinterpret_cast<float3*>(s_pfwd + INC_FLOATS);
    float* s_env = s_pfwd + INC_FLOATS + (IS ? 0 : sample_table_floats(a.N));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & (PIX_G - 1), grp = lane / PIX_G;
    float* sinc = s_pfwd + (warp * PIX_GPW + grp) * SHADE_INC_STRIDE;
    if constexpr (IS) smp.t = EnvTable(smp.table);
    else for (int i = threadIdx.x; i < a.N; i += SHADE_THREADS) s_smp[i] = fib_sample(i, a.N);
    if (SMEM_ENV)
        for (int i = threadIdx.x; i < (FILT ? lv.total : a.He * a.We) * 3; i += SHADE_THREADS) s_env[i] = a.env[i];
    __syncthreads();
    const float* env = SMEM_ENV ? s_env : a.env;
    const float invN = 1.0f / (float)a.N;
    const size_t HW = (size_t)a.P, total = (size_t)pv.V * HW;
    const size_t units = (total + PIX_GPW - 1) / PIX_GPW;
    for (size_t u = (size_t)blockIdx.x * SHADE_WARPS + warp; u < units; u += (size_t)gridDim.x * SHADE_WARPS) {
        const size_t p_raw = u * PIX_GPW + grp;
        const bool valid = p_raw < total;
        const size_t vq = valid ? p_raw : total - 1;   // idle groups of the last warp shade a copy, write nothing
        const int v = (int)(vq / HW);
        const size_t q = vq - (size_t)v * HW;
        const bool live = valid && (!pv.mask || pv.mask[vq]);
        GaussianOperands o;
        float3 nh;
        load_pixel(a, pv, v, q, o, nh);
        stage_pixel_incidents(a, v, q, sinc, sub);
        const float* tr = view_transform(a, pv, v);
        const float* vis_row = a.visibility + (size_t)v * a.N * HW + q;
        float pbr[3] = {0, 0, 0}, spec[3] = {0, 0, 0}, diff[3] = {0, 0, 0}, mv = 0;
        if (live) {
            GgxFrame f{};
            if constexpr (IS) f = pixel_ggx_frame(a, pv, smp, v, q, o, nh);
            for (int i = sub; i < a.N; i += PIX_G) {
                float3 d;
                float ar = PIX_AREA;
                if constexpr (IS) d = importance_sample(smp, (uint32_t)q, i, nh, f, ar);
                else d = rotate_from_z(nh.x, nh.y, nh.z, s_smp[i]);
                const float vis = vis_row[(size_t)i * HW];
                SampleEvalT<FILT> e;
                eval_env_any<SMEM_ENV>(tr, env, a, lv, ar * invN, d.x, d.y, d.z, vis, e);
                pixel_local(a, o, sinc, d, e);
                eval_ggx<false>(o.V, o.Ns, o, d.x, d.y, d.z, e);
#pragma unroll
                for (int c = 0; c < 3; ++c) {                 // the per-Gaussian forward's expressions
                    const float loc = fmaxf(e.local_raw[c], 0.f);
                    const float Lc = loc + e.glob[c];
                    const float T = Lc * ar * e.ndi;
                    const float fd = o.base[c] / PI_F;
                    pbr[c] += (fd + e.fs) * T; spec[c] += e.fs * T; diff[c] += T;
                }
                mv += vis;
            }
        }
        __syncwarp();
#pragma unroll
        for (int c = 0; c < 3; ++c) { pbr[c] = group_sum<PIX_G>(pbr[c]); spec[c] = group_sum<PIX_G>(spec[c]); diff[c] = group_sum<PIX_G>(diff[c]); }
        mv = group_sum<PIX_G>(mv);
        if (sub == 0 && valid) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const size_t k = (3 * (size_t)v + c) * HW + q;
                a.pbr[k] = live ? pbr[c] * invN : 0.f;
                a.specular[k] = live ? spec[c] * invN : 0.f;
                a.diffuse[k] = live ? diff[c] * invN : 0.f;
            }
            a.mean_vis[vq] = live ? mv * invN : 0.f;
        }
    }
}

// Backward: the per-Gaussian backward's per-sample code (ENV_MODE <= ENV_CAS or deterministic: no warp collectives
// inside the sample loop, so masked groups skip it).  3 resident CTAs (<= 168 registers): at 4 (128) every
// mode but the deterministic ones spills a few words.  dL/dbase, dL/droughness and dL/dincidents are written per pixel
// (zeros for masked ones), dL/denv is accumulated over every view.
template <int ENV_MODE, bool FILT, bool IS>
__global__ void __launch_bounds__(SHADE_THREADS, 3)
pixel_shade_bwd_kernel(const ShadeArgs a, const PixelView pv, const EnvLevels lv, ImportanceSampler smp) {
    static_assert(ENV_MODE != ENV_TAG, "the tagged mode's collectives need a warp-uniform sample loop");
    // [incident slots][SH-gradient accumulators][sample table][env ...]
    extern __shared__ __align__(16) float s_pbwd[];
    constexpr bool SMEM_ENV = EnvGrad<ENV_MODE>::SMEM_ENV;
    constexpr int INC_FLOATS = SHADE_WARPS * PIX_GPW * SHADE_INC_STRIDE;
    constexpr int DINC_FLOATS = 48 * SHADE_THREADS;
    constexpr int RQ = 48 / PIX_G;                      // finished SH-gradient components per lane
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & (PIX_G - 1), grp = lane / PIX_G;
    float* sinc = s_pbwd + (warp * PIX_GPW + grp) * SHADE_INC_STRIDE;
    float4* acc4 = reinterpret_cast<float4*>(s_pbwd + INC_FLOATS) + threadIdx.x;
    float3* s_smp = reinterpret_cast<float3*>(s_pbwd + INC_FLOATS + DINC_FLOATS);
    if constexpr (IS) smp.t = EnvTable(smp.table);
    else for (int i = threadIdx.x; i < a.N; i += SHADE_THREADS) s_smp[i] = fib_sample(i, a.N);
    EnvGrad<ENV_MODE> eg(a, s_pbwd + INC_FLOATS + DINC_FLOATS + (IS ? 0 : sample_table_floats(a.N)), warp, FILT ? lv.total : a.He * a.We);
    __syncthreads();                                     // the sample table (EnvGrad syncs only in its shared-memory modes)
    const float invN = 1.0f / (float)a.N;
    const size_t HW = (size_t)a.P, total = (size_t)pv.V * HW;
    const size_t units = (total + PIX_GPW - 1) / PIX_GPW;
    for (size_t u = (size_t)blockIdx.x * SHADE_WARPS + warp; u < units; u += (size_t)gridDim.x * SHADE_WARPS) {
        const size_t p_raw = u * PIX_GPW + grp;
        const bool valid = p_raw < total;
        const size_t vq = valid ? p_raw : total - 1;
        const int v = (int)(vq / HW);
        const size_t q = vq - (size_t)v * HW;
        const bool live = valid && (!pv.mask || pv.mask[vq]);
        GaussianOperands o;
        float3 nh;
        load_pixel(a, pv, v, q, o, nh);
        stage_pixel_incidents(a, v, q, sinc, sub);
        const float* tr = view_transform(a, pv, v);
        const float* vis_row = a.visibility + (size_t)v * a.N * HW + q;
        float gp[3], gs[3], gd[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const size_t k = (3 * (size_t)v + c) * HW + q;
            gp[c] = a.g_pbr[k] * invN;
            gs[c] = a.g_specular ? a.g_specular[k] * invN : 0.f;
            gd[c] = a.g_diffuse ? a.g_diffuse[k] * invN : 0.f;
        }
        float dbase[3] = {0, 0, 0}, drough = 0.f, dV[3] = {0, 0, 0};
#pragma unroll
        for (int k = 0; k < 12; ++k) acc4[k * SHADE_THREADS] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live) {
            GgxFrame f{};
            if constexpr (IS) f = pixel_ggx_frame(a, pv, smp, v, q, o, nh);
            for (int i = sub; i < a.N; i += PIX_G) {
                float3 d;
                float ar = PIX_AREA;
                if constexpr (IS) d = importance_sample(smp, (uint32_t)q, i, nh, f, ar);
                else d = rotate_from_z(nh.x, nh.y, nh.z, s_smp[i]);
                const float vis = vis_row[(size_t)i * HW];
                SampleEvalT<FILT> e;
                eval_env_any<SMEM_ENV>(tr, eg.env, a, lv, ar * invN, d.x, d.y, d.z, vis, e);
                pixel_local(a, o, sinc, d, e);
                eval_ggx<true>(o.V, o.Ns, o, d.x, d.y, d.z, e);
                float dfs = 0.f;
                float dG[3], dLg[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) {                 // the per-Gaussian backward's expressions
                    const float loc = fmaxf(e.local_raw[c], 0.f);
                    const float T = (loc + e.glob[c]) * ar * e.ndi;
                    const float fd = o.base[c] * INV_PI_F;
                    const float dT = gp[c] * (fd + e.fs) + gs[c] * e.fs + gd[c];
                    dbase[c] += gp[c] * T * INV_PI_F; dfs += (gp[c] + gs[c]) * T;
                    const float dL = dT * ar * e.ndi;
                    dLg[c] = e.local_raw[c] >= 0.f ? dL : 0.f;      // clamp_min(0) passes the gradient at equality
                    dG[c] = dL * vis;                                // -> env texels (grid_sample backward)
                }
                if (a.incidents) accumulate_dinc(acc4, dLg, e.w);
                eg.scatter(a, e.taps, dG, lane);
                ggx_backward(o.V, o.Ns, o, e, dfs, drough, dV);
            }
        }
        __syncwarp();
        // ---- group reduction and per-pixel outputs ---------------------------------------------
#pragma unroll
        for (int c = 0; c < 3; ++c) dbase[c] = group_sum<PIX_G>(dbase[c]);
        drough = group_sum<PIX_G>(drough);
        if (a.incidents) {
            float dinc[48];
#pragma unroll
            for (int k = 0; k < 12; ++k) { const float4 t = acc4[k * SHADE_THREADS]; dinc[4 * k] = t.x; dinc[4 * k + 1] = t.y; dinc[4 * k + 2] = t.z; dinc[4 * k + 3] = t.w; }
            group_reduce_scatter<PIX_G, 48>(dinc, sub);   // lane `sub` now owns components [sub*RQ, sub*RQ + RQ)
            if (valid) {
#pragma unroll
                for (int k = 0; k < RQ; ++k) a.d_incidents[(48 * (size_t)v + sub * RQ + k) * HW + q] = dinc[k];
            }
        }
        if (valid && sub == 0) {
#pragma unroll
            for (int c = 0; c < 3; ++c) a.d_base[(3 * (size_t)v + c) * HW + q] = dbase[c];
            a.d_rough[vq] = drough;
        }
    }
    eg.flush(a);
}

static size_t pixel_fixed_bytes(int N, bool is) {
    return (size_t)SHADE_WARPS * PIX_GPW * SHADE_INC_STRIDE * sizeof(float) + (is ? 0 : (size_t)sample_table_floats(N) * sizeof(float));
}

static int pixel_units(const PixelView& pv, const ShadeArgs& a) { return (int)(((size_t)pv.V * a.P + PIX_GPW - 1) / PIX_GPW); }

static int launch_pixel_forward(ShadeArgs a, const PixelView& pv, const EnvLevels& lv, bool filt, const ImportanceSampler& smp,
                                cudaStream_t stream) {
    const size_t env_bytes = env_texels(a, lv, filt) * 3 * sizeof(float);
    const bool smem_env = env_bytes <= 40 * 1024;       // as the per-Gaussian forward
    a.env_in_smem = smem_env;
    const bool is = smp.table != nullptr;
    const size_t smem = pixel_fixed_bytes(a.N, is) + (smem_env ? env_bytes : 0);
    const int units = pixel_units(pv, a), sms = num_sms();
    const auto go = [&](auto k) { return shade_launch(k, a, units, sms, smem, stream, pv, lv, smp); };
    if (is) {
        if (filt) return smem_env ? go(pixel_shade_fwd_kernel<true, true, true>) : go(pixel_shade_fwd_kernel<false, true, true>);
        return smem_env ? go(pixel_shade_fwd_kernel<true, false, true>) : go(pixel_shade_fwd_kernel<false, false, true>);
    }
    if (filt) return smem_env ? go(pixel_shade_fwd_kernel<true, true, false>) : go(pixel_shade_fwd_kernel<false, true, false>);
    return smem_env ? go(pixel_shade_fwd_kernel<true, false, false>) : go(pixel_shade_fwd_kernel<false, false, false>);
}

// the env-gradient mode as the per-Gaussian backward picks it at its default highest mode
static int launch_pixel_backward(ShadeArgs a, const PixelView& pv, const EnvLevels& lv, bool filt, const ImportanceSampler& smp,
                                 cudaStream_t stream) {
    const int sms = num_sms();
    return shade_backward(a, pv.V, ENV_CAS, env_texels(a, lv, filt), sms, stream, [&](auto mode, const ShadeArgs& x, size_t env_smem) {
        constexpr int M = decltype(mode)::value;
        if constexpr (M == ENV_TAG) return (int)R3DG_ERR_UNSUPPORTED;     // above the cap: never selected
        else {
            const bool is = smp.table != nullptr;
            const size_t smem = pixel_fixed_bytes(x.N, is) + (size_t)48 * SHADE_THREADS * sizeof(float) + env_smem;
            const int units = pixel_units(pv, x);
            const auto go = [&](auto k) { return shade_launch(k, x, units, sms, smem, stream, pv, lv, smp); };
            if (is) return filt ? go(pixel_shade_bwd_kernel<M, true, true>) : go(pixel_shade_bwd_kernel<M, false, true>);
            return filt ? go(pixel_shade_bwd_kernel<M, true, false>) : go(pixel_shade_bwd_kernel<M, false, false>);
        }
    });
}

}  // namespace r3dg

// ---- C ABI --------------------------------------------------------------------------------------
using namespace r3dg;
extern "C" {

// the shared checks of both directions; ShadeArgs and PixelView of the call
static int pixel_args(const r3dg_pixel_args* s, ShadeArgs& a, PixelView& pv, ImportanceSampler& smp) {
    if (!s || s->V < 1 || s->V > R3DG_MAX_VIEWS || s->H < 1 || s->W < 1 || s->N < 1 || s->env_h < 1 || s->env_w < 1)
        return R3DG_ERR_BAD_ARG;
    if (!s->base_color || !s->roughness || !s->normal || !s->points || !s->campos || !s->env || !s->visibility)
        return R3DG_ERR_BAD_ARG;
    if (s->transform_per_view && !s->env_transform) return R3DG_ERR_BAD_ARG;
    if ((size_t)s->N * sizeof(float3) > BAKE_SAMPLE_SMEM) return R3DG_ERR_UNSUPPORTED;
    if ((long long)s->V * s->H * s->W > 0x7fffffffLL) return R3DG_ERR_UNSUPPORTED;
    if (s->sampler_table && (s->n_env < 0 || s->n_ggx < 0 || (long long)s->N - s->n_env - s->n_ggx < 1)) return R3DG_ERR_BAD_ARG;
    smp = ImportanceSampler{};
    if (s->sampler_table) {
        smp.table = s->sampler_table; smp.T = s->sampler_transform;
        smp.N = s->N; smp.n_env = s->n_env; smp.n_ggx = s->n_ggx; smp.seed = s->seed;
    }
    a = ShadeArgs{};
    a.P = s->H * s->W; a.N = s->N; a.He = s->env_h; a.We = s->env_w;
    a.base_color = s->base_color; a.roughness = s->roughness; a.normals = s->normal; a.incidents = s->incidents;
    a.env = s->env; a.transform = s->env_transform; a.visibility = s->visibility;
    a.pbr = s->pbr; a.diffuse = s->diffuse_light; a.specular = s->specular; a.mean_vis = s->mean_visibility;
    a.g_pbr = s->dL_dpbr; a.g_diffuse = s->dL_ddiffuse_light; a.g_specular = s->dL_dspecular;
    a.d_base = s->dL_dbase_color; a.d_rough = s->dL_droughness; a.d_incidents = s->dL_dincidents; a.d_env = s->dL_denv;
    a.det = DetAcc{nullptr, nullptr, 0};
    pv = PixelView{s->V, s->transform_per_view != 0, s->points, s->campos, s->mask};
    return 0;
}

int r3dg_shade_pixels_forward(const r3dg_pixel_args* s, r3dg_stream_t stream) {
    ShadeArgs a;
    PixelView pv;
    ImportanceSampler smp;
    const int rc = pixel_args(s, a, pv, smp);
    if (rc) return rc;
    if (!a.pbr || !a.diffuse || !a.specular || !a.mean_vis) return R3DG_ERR_BAD_ARG;
    const EnvLevels lv = env_levels(a.He, a.We);
    const bool filt = s->env_pyramid && lv.L > 1;
    if (filt) a.env = s->env_pyramid;
    return launch_pixel_forward(a, pv, lv, filt, smp, (cudaStream_t)stream);
}

int r3dg_shade_pixels_backward(const r3dg_pixel_args* s, r3dg_stream_t stream) {
    ShadeArgs a;
    PixelView pv;
    ImportanceSampler smp;
    int rc = pixel_args(s, a, pv, smp);
    if (rc) return rc;
    if (!a.g_pbr || !a.d_base || !a.d_rough || !a.d_env || (a.incidents && !a.d_incidents)) return R3DG_ERR_BAD_ARG;
    if (s->env_pyramid && !s->dL_denv_pyramid) return R3DG_ERR_BAD_ARG;
    const EnvLevels lv = env_levels(a.He, a.We);
    const bool filt = s->env_pyramid && lv.L > 1;
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
    rc = launch_pixel_backward(a, pv, lv, filt, smp, st);
    if (rc || !filt) return rc;
    return launch_env_pyramid_adjoint(lv, a.d_env, d_env, st);               // dL/denv through the pyramid
}

}  // extern "C"
