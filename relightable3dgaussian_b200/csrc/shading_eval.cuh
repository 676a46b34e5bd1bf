// The shading step's per-sample pieces, shared by the per-Gaussian kernels (shading.cu) and the per-pixel ones
// (pixel_shading.cu): the argument record, the SH basis, the environment taps (point and filtered), the sample record
// with its light evaluation, the group reductions, the env-gradient accumulation modes and the backward's launch
// policy.  Both files are compiled with -fmad=false, so each op rounds as its PyTorch counterpart does.
#pragma once
#include <algorithm>
#include <type_traits>
#include "brdf.cuh"
#include "common.cuh"
#include "detacc.cuh"
#include "envfilter.cuh"
#include "kernels.h"

namespace r3dg {

#define SHADE_THREADS 128
#define SHADE_WARPS (SHADE_THREADS / 32)

struct ShadeArgs {
    int P, N, He, We, env_in_smem;
    const float *base_color, *roughness, *normals, *viewdirs, *incidents, *env, *transform;
    const float *visibility, *dirs, *areas;
    // forward outputs
    float *pbr, *diffuse, *specular, *mean_lights, *mean_local, *mean_global, *mean_vis;
    float *s_lights, *s_local, *s_global;        // optional per-sample [P,N,3]
    // backward
    const float *g_pbr, *g_diffuse, *g_specular;
    float *d_base, *d_rough, *d_view, *d_incidents, *d_env;
    DetAcc det;                                  // deterministic mode: dL/denv accumulators [He * We * 3] (detacc.cuh)
    uint32_t* det_scale;                         // deterministic mode: the call's scale word, behind the accumulators
};

__device__ __forceinline__ void sh_basis3(float x, float y, float z, float* w) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    w[0] = 0.28209479177387814f;
    w[1] = -0.4886025119029199f * y; w[2] = 0.4886025119029199f * z; w[3] = -0.4886025119029199f * x;
    w[4] = 1.0925484305920792f * xy; w[5] = -1.0925484305920792f * yz; w[6] = 0.31539156525252005f * (2.0f * zz - xx - yy);
    w[7] = -1.0925484305920792f * xz; w[8] = 0.5462742152960396f * (xx - yy);
    w[9] = -0.5900435899266435f * y * (3.f * xx - yy); w[10] = 2.890611442640554f * xy * z;
    w[11] = -0.4570457994644658f * y * (4.f * zz - xx - yy); w[12] = 0.3731763325901154f * z * (2.f * zz - 3.f * xx - 3.f * yy);
    w[13] = -0.4570457994644658f * x * (4.f * zz - xx - yy); w[14] = 1.445305721320277f * z * (xx - yy);
    w[15] = -0.5900435899266435f * x * (xx - 3.f * yy);
}

template <int K> struct EnvTaps { int idx[K]; float w[K]; };   // texel base offsets (float index of channel 0, or -1) + weights
using EnvTap = EnvTaps<4>;

// the filtered mode's grid_sample coordinates of dir d in [0, 1]: u along the columns, v along the rows
__device__ __forceinline__ void env_uv(float dx, float dy, float dz, float& u, float& v) {
    const float phi = acosf(dz) - 1e-6f;
    const float theta = atan2f(dy, dx);
    const float qy = (phi / PI_F) * 2.0f - 1.0f;
    const float qx = -theta / PI_F;
    u = (qx + 1.0f) / 2.0f;
    v = (qy + 1.0f) / 2.0f;
}

// the four bilinear taps of (u, v) on an He x We texture, into taps B .. B+3 of t
template <int B, int K>
__device__ __forceinline__ void fill_taps(float u, float v, int He, int We, EnvTaps<K>& t) {
    const float ix = u * (float)(We - 1);
    const float iy = v * (float)(He - 1);
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float ax = ix - fx, ay = iy - fy;        // == ix - ix_nw ; (ix_se - ix) == 1 - ax
    const int xs[2] = {x0, x0 + 1}, ys[2] = {y0, y0 + 1};
    const float wx[2] = {(fx + 1.0f) - ix, ax}, wy[2] = {(fy + 1.0f) - iy, ay};
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const bool in = xs[i] >= 0 && xs[i] < We && ys[j] >= 0 && ys[j] < He;
            t.idx[B + 2 * j + i] = in ? (ys[j] * We + xs[i]) * 3 : -1;
            t.w[B + 2 * j + i] = wx[i] * wy[j];
        }
}

// grid_sample(bilinear, zeros padding, align_corners=True) at the lat-long coordinates of dir d (the point lookup; the
// filtered mode's taps below repeat its arithmetic through env_uv and fill_taps)
__device__ __forceinline__ EnvTap env_taps(float dx, float dy, float dz, int He, int We) {
    const float phi = acosf(dz) - 1e-6f;
    const float theta = atan2f(dy, dx);
    const float qy = (phi / PI_F) * 2.0f - 1.0f;
    const float qx = -theta / PI_F;
    const float ix = ((qx + 1.0f) / 2.0f) * (float)(We - 1);
    const float iy = ((qy + 1.0f) / 2.0f) * (float)(He - 1);
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy;
    const float ax = ix - fx, ay = iy - fy;        // == ix - ix_nw ; (ix_se - ix) == 1 - ax
    EnvTap t;
    const int xs[2] = {x0, x0 + 1}, ys[2] = {y0, y0 + 1};
    const float wx[2] = {(fx + 1.0f) - ix, ax}, wy[2] = {(fy + 1.0f) - iy, ay};
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const bool in = xs[i] >= 0 && xs[i] < We && ys[j] >= 0 && ys[j] < He;
            t.idx[2 * j + i] = in ? (ys[j] * We + xs[i]) * 3 : -1;
            t.w[2 * j + i] = wx[i] * wy[j];
        }
    return t;
}

// The filtered lookup (include/r3dg_b200.h, "PREFILTERED ENVIRONMENT"): the trilinear taps of d on the pyramid `lv`
// for a sample of solid angle omega.  lambda = log2(omega / Omega0(theta)) / 2, clamped to [0, L-1], is evaluated in
// fp32; at lambda <= 0 the taps are env_taps' four, weights and order unchanged (the upper four are absent).
__device__ __forceinline__ EnvTaps<8> env_taps_filtered(float dx, float dy, float dz, const EnvLevels& lv, float omega) {
    float u, v;
    env_uv(dx, dy, dz, u, v);
    const float st = sqrtf(fmaxf(1.0f - dz * dz, 0.0f));
    const float lam = fminf(fmaxf(0.5f * log2f(omega / (lv.dtdp * fmaxf(st, lv.sin_half))), 0.0f), (float)(lv.L - 1));
    const int l0 = (int)lam;
    const float f = lam - (float)l0;
    EnvTaps<8> t;
    fill_taps<0>(u, v, lv.h[l0], lv.w[l0], t);
    const int o0 = 3 * lv.off[l0];
#pragma unroll
    for (int q = 0; q < 4; ++q) { if (t.idx[q] >= 0) t.idx[q] += o0; t.w[q] *= 1.0f - f; }
    if (f > 0.0f) {
        fill_taps<4>(u, v, lv.h[l0 + 1], lv.w[l0 + 1], t);
        const int o1 = 3 * lv.off[l0 + 1];
#pragma unroll
        for (int q = 4; q < 8; ++q) { if (t.idx[q] >= 0) t.idx[q] += o1; t.w[q] *= f; }
    } else {
#pragma unroll
        for (int q = 4; q < 8; ++q) { t.idx[q] = -1; t.w[q] = 0.0f; }
    }
    return t;
}

#define SHADE_INC_STRIDE 52       // floats per group slot: 16-byte aligned, bank-staggered (52 mod 32 = 20)

template <bool FILT = false>
struct SampleEvalT {      // forward quantities of one (Gaussian, direction) pair; FILT: the filtered mode's 8 env taps
    float local_raw[3], glob[3], ndi, fs;
    float w[16];
    EnvTaps<FILT ? 8 : 4> taps;
    // GGX intermediates for the backward
    float H[3], hn, NoL, NoV, NoH, VoH, NoL_r, NoV_r, NoH_r, VoH_r, p2, frac0, nom0, nom1, nom2, nom_r, nom;
};
using SampleEval = SampleEvalT<false>;

// Each sample's evaluation comes in three parts, so that the view kernels can run the first two once for all views:
// the environment light (depends on the env transform), the local SH light and n.w (depend on the Gaussian only),
// and GGX_specular (depends on the view).
// the global light env(T d) * vis and its texel taps; T: the [3,3] env transform or NULL
template <bool SMEM_ENV>
__device__ __forceinline__ void eval_env(const float* T, const float* __restrict__ env, int He, int We, float dx, float dy,
                                         float dz, float vis, SampleEval& e) {
    float ex = dx, ey = dy, ez = dz;
    if (T) {                                               // dirs @ transform.T  (scene/envmap.py:39-42)
        // the sums start from +0 like a BLAS product: a row of -0 terms gives +0 (not -0), which decides the env
        // column at the seam (atan2(+0, x < 0) = +pi -> column 0, atan2(-0, x < 0) = -pi -> column We-1)
        ex = 0.f + dx * T[0] + dy * T[1] + dz * T[2]; ey = 0.f + dx * T[3] + dy * T[4] + dz * T[5]; ez = 0.f + dx * T[6] + dy * T[7] + dz * T[8];
    }
    e.taps = env_taps(ex, ey, ez, He, We);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float s = 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t) if (e.taps.idx[t] >= 0) s += (SMEM_ENV ? env[e.taps.idx[t] + c] : __ldg(env + e.taps.idx[t] + c)) * e.taps.w[t];
        e.glob[c] = s * vis;
    }
}

// the filtered mode's global light: env is the pyramid, omega the sample's solid angle
template <bool SMEM_ENV>
__device__ __forceinline__ void eval_env_filtered(const float* T, const float* __restrict__ env, const EnvLevels& lv, float omega,
                                                  float dx, float dy, float dz, float vis, SampleEvalT<true>& e) {
    float ex = dx, ey = dy, ez = dz;
    if (T) { ex = 0.f + dx * T[0] + dy * T[1] + dz * T[2]; ey = 0.f + dx * T[3] + dy * T[4] + dz * T[5]; ez = 0.f + dx * T[6] + dy * T[7] + dz * T[8]; }
    e.taps = env_taps_filtered(ex, ey, ez, lv, omega);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float s = 0.f;
#pragma unroll
        for (int t = 0; t < 8; ++t) if (e.taps.idx[t] >= 0) s += (SMEM_ENV ? env[e.taps.idx[t] + c] : __ldg(env + e.taps.idx[t] + c)) * e.taps.w[t];
        e.glob[c] = s * vis;
    }
}

// the global light of either mode (omega = area / N: read by the filtered mode only)
template <bool SMEM_ENV, bool FILT>
__device__ __forceinline__ void eval_env_any(const float* T, const float* __restrict__ env, const ShadeArgs& a, const EnvLevels& lv,
                                             float omega, float dx, float dy, float dz, float vis, SampleEvalT<FILT>& e) {
    if constexpr (FILT) eval_env_filtered<SMEM_ENV>(T, env, lv, omega, dx, dy, dz, vis, e);
    else eval_env<SMEM_ENV>(T, env, a.He, a.We, dx, dy, dz, vis, e);
}

// the local SH light (before its clamp) and n.w with the raw normal
template <bool INC_SMEM, class E>
__device__ __forceinline__ void eval_local(const GaussianOperands& o, const float* __restrict__ sinc, float dx, float dy, float dz,
                                           E& e) {
    sh_basis3(dx, dy, dz, e.w);
    if (INC_SMEM) {
        float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int q = 0; q < 12; ++q) {
            const float4 v = reinterpret_cast<const float4*>(sinc)[q];
            const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[(4 * q + j) % 3] += e.w[(4 * q + j) / 3] * vv[j];   // per channel still k = 0..15 in order
            if (q % 3 == 2) asm volatile("" ::: "memory");     // keep at most 3 LDS.128 in flight: hoisting all 12 costs the 48 registers back
        }
        e.local_raw[0] = acc[0]; e.local_raw[1] = acc[1]; e.local_raw[2] = acc[2];
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < 16; ++k) s += e.w[k] * o.inc[3 * k + c];      // eval_sh's left-to-right order
            e.local_raw[c] = s;
        }
    }
    e.ndi = fmaxf(o.n[0] * dx + o.n[1] * dy + o.n[2] * dz, 0.f);
}

// ---- sub-warp groups ---------------------------------------------------------------------------
// A group of G lanes (G = 8, 16 or 32) owns one Gaussian, so a warp shades 32/G Gaussians at once:
// at the training sample counts (N = 32 / 64, script/run_*.sh) a whole warp per Gaussian leaves each
// lane 1-2 samples and the per-Gaussian work (operand loads, 58 values x 5 shuffle levels in the
// backward) dominates.  Groups read consecutive rows of the baked tensors, so loads stay coalesced.
template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Transposed butterfly ("reduce-scatter") over the G lanes of a group: V values per lane in, and
// lane `sub` returns with v[0 .. V/G) = the group totals of components [sub*V/G, (sub+1)*V/G).
// V*(1 - 1/G) shuffles instead of V*log2(G).
template <int G, int V>
__device__ __forceinline__ void group_reduce_scatter(float (&v)[V], int sub) {
    static_assert(V % G == 0, "V must be a multiple of the group width");
    int n = V;
#pragma unroll
    for (int m = G / 2; m > 0; m >>= 1) {
        const bool upper = (sub & m) != 0;
        const int h = n / 2;
#pragma unroll
        for (int i = 0; i < V / 2; ++i) {
            if (i < h) {
                const float send = upper ? v[i] : v[i + h];
                const float keep = upper ? v[i + h] : v[i];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, m);
            }
        }
        n = h;
    }
}

// ---- environment-map gradient (grid_sample backward: a scatter-add of P*N*4 taps) ----------------
// There is no native fp32 shared-memory atomic add on sm_90: `atomicAdd(float*)` on shared memory
// compiles to an LDS / FADD / ATOMS.CAST.SPIN loop that occupies the LSU for many cycles per warp
// instruction, and 12 of them per sample bounded the whole backward kernel.  ENV_TAG mode gives
// every warp a PRIVATE float4 {r,g,b,-} copy of the texture gradient and resolves the (rare)
// intra-warp collisions with a one-byte tag per texel: every pending lane stores its lane id, the
// id that survives owns the texel this round and does a plain 128-bit read-modify-write, the losers
// retry.  The copies are summed and flushed once per CTA.
// The deterministic mode accumulates every tap through the fixed-point primitive (detacc.cuh): ENV_DET_SMEM into
// per-CTA integer accumulators in shared memory whose words are added to the global ones once per CTA (integer sums,
// so the flush order does not matter either), ENV_DET_GLOBAL straight into the global accumulators (larger textures).
// Every tap is linear in the call's cotangents dL_dpbr, dL_ddiffuse_light and dL_dspecular; its fixed point is scaled
// by the exponent of their largest magnitude (det_scale_kernel), one exponent per call.
enum { ENV_GLOBAL = 0, ENV_CAS = 1, ENV_TAG = 2, ENV_DET_SMEM = 3, ENV_DET_GLOBAL = 4 };

__device__ __forceinline__ void warp_private_add(float4* wg, volatile unsigned char* tag, int texel, float x, float y, float z, int lane) {
    bool pending = texel >= 0;
    while (true) {                                   // warp-uniform trip count
        if (pending) tag[texel] = (unsigned char)lane;
        __syncwarp();
        if (pending && tag[texel] == (unsigned char)lane) {
            float4 acc = wg[texel];
            acc.x += x; acc.y += y; acc.z += z;
            wg[texel] = acc;
            pending = false;
        }
        __syncwarp();
        if (!__any_sync(0xffffffffu, pending)) break;
    }
}

// The env-gradient state of one backward CTA in its shared memory `s_mem`: the constructor stages the texture and
// zeroes the accumulators of ENV_MODE, scatter() adds one sample's taps, flush() adds the CTA's total to dL/denv.
template <int ENV_MODE>
struct EnvGrad {
    static constexpr bool SMEM_ENV = ENV_MODE != ENV_GLOBAL && ENV_MODE != ENV_DET_GLOBAL;
    int nt, ne, nflag, det_e;
    float *s_env, *s_genv;
    float4 *wgrad_all, *wgrad;
    volatile unsigned char* wtag;
    uint64_t* s_dwords;
    uint32_t* s_dflags;
    const float* env;                                // the texture the samples read (shared or global memory)
    float* genv;                                     // ENV_CAS / ENV_GLOBAL: where the taps are added

    // bytes of `s_mem` the constructor lays out for a texture of nt texels (0 for the global-memory modes):
    // ENV_CAS: [env ne][grad ne]; ENV_TAG: [env ne (padded to 4)][per warp: float4 grad[nt]][per warp: tag[nt] padded to 16];
    // ENV_DET_SMEM: [env ne (padded to 2)][accumulator words 3 ne][flag words (ne + 15) / 16]
    static __host__ __device__ size_t smem_bytes(size_t nt) {
        const size_t ne = nt * 3;
        if (ENV_MODE == ENV_CAS) return 2 * ne * sizeof(float);
        if (ENV_MODE == ENV_TAG) return ((ne + 3) & ~(size_t)3) * sizeof(float) + SHADE_WARPS * (nt * sizeof(float4) + ((nt + 15) & ~(size_t)15));
        if (ENV_MODE == ENV_DET_SMEM) return ((ne + 1) & ~(size_t)1) * sizeof(float) + 3 * ne * sizeof(uint64_t) + (ne + 15) / 16 * sizeof(uint32_t);
        return 0;
    }

    // texels: of the texture the samples read (He * We, or every level of the filtered mode's pyramid)
    __device__ __forceinline__ EnvGrad(const ShadeArgs& a, float* s_mem, int warp, int texels) {
        nt = texels; ne = nt * 3;
        s_env = s_mem;
        s_genv = s_mem + ne;
        const int ne4 = (ne + 3) & ~3, ntp = (nt + 15) & ~15;
        wgrad_all = reinterpret_cast<float4*>(s_mem + ne4);
        wgrad = wgrad_all + (size_t)warp * nt;
        wtag = reinterpret_cast<unsigned char*>(wgrad_all + (size_t)SHADE_WARPS * nt) + (size_t)warp * ntp;
        s_dwords = reinterpret_cast<uint64_t*>(s_mem + ((ne + 1) & ~1));
        s_dflags = reinterpret_cast<uint32_t*>(s_dwords + 3 * (size_t)ne);
        nflag = (ne + 15) >> 4;
        det_e = ENV_MODE == ENV_DET_SMEM || ENV_MODE == ENV_DET_GLOBAL ? det_scale_exp(*a.det_scale) : 0;
        if (SMEM_ENV) {
            for (int i = threadIdx.x; i < ne; i += SHADE_THREADS) s_env[i] = a.env[i];
            if (ENV_MODE == ENV_CAS) for (int i = threadIdx.x; i < ne; i += SHADE_THREADS) s_genv[i] = 0.f;
            if (ENV_MODE == ENV_TAG) for (int i = threadIdx.x; i < SHADE_WARPS * nt; i += SHADE_THREADS) wgrad_all[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ENV_MODE == ENV_DET_SMEM) {
                for (int i = threadIdx.x; i < 3 * ne; i += SHADE_THREADS) s_dwords[i] = 0u;
                for (int i = threadIdx.x; i < nflag; i += SHADE_THREADS) s_dflags[i] = 0u;
            }
            __syncthreads();
        }
        env = SMEM_ENV ? s_env : a.env;
        genv = ENV_MODE == ENV_CAS ? s_genv : a.d_env;
    }

    // dG: the sample's light cotangent times its visibility (zero for an inactive lane); called by every lane of the warp
    template <int K>
    __device__ __forceinline__ void scatter(const ShadeArgs& a, const EnvTaps<K>& taps, const float* dG, int lane) {
        if (ENV_MODE == ENV_TAG) {
            const bool any = dG[0] != 0.f || dG[1] != 0.f || dG[2] != 0.f;
#pragma unroll
            for (int t = 0; t < K; ++t) {
                const int texel = (any && taps.idx[t] >= 0) ? taps.idx[t] / 3 : -1;
                warp_private_add(wgrad, wtag, texel, dG[0] * taps.w[t], dG[1] * taps.w[t], dG[2] * taps.w[t], lane);
            }
        } else if (ENV_MODE == ENV_DET_SMEM || ENV_MODE == ENV_DET_GLOBAL) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                if (dG[c] != 0.f) {
#pragma unroll
                    for (int t = 0; t < K; ++t)
                        if (taps.idx[t] >= 0) {
                            if (ENV_MODE == ENV_DET_SMEM) det_add(s_dwords, s_dflags, ne, taps.idx[t] + c, dG[c] * taps.w[t], det_e, true);
                            else det_add(a.det, taps.idx[t] + c, dG[c] * taps.w[t], det_e);
                        }
                }
        } else {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                if (dG[c] != 0.f) {
#pragma unroll
                    for (int t = 0; t < K; ++t) if (taps.idx[t] >= 0) atomicAdd(genv + taps.idx[t] + c, dG[c] * taps.w[t]);
                }
        }
    }

    __device__ __forceinline__ void flush(const ShadeArgs& a) {
        if (ENV_MODE == ENV_CAS) {
            __syncthreads();
            for (int i = threadIdx.x; i < ne; i += SHADE_THREADS) { const float v = s_genv[i]; if (v != 0.f) atomicAdd(a.d_env + i, v); }
        }
        if (ENV_MODE == ENV_TAG) {
            __syncthreads();
            for (int t = threadIdx.x; t < nt; t += SHADE_THREADS) {
                float4 s = wgrad_all[t];
#pragma unroll
                for (int w = 1; w < SHADE_WARPS; ++w) { const float4 v = wgrad_all[(size_t)w * nt + t]; s.x += v.x; s.y += v.y; s.z += v.z; }
                if (s.x != 0.f) atomicAdd(a.d_env + 3 * t, s.x);
                if (s.y != 0.f) atomicAdd(a.d_env + 3 * t + 1, s.y);
                if (s.z != 0.f) atomicAdd(a.d_env + 3 * t + 2, s.z);
            }
        }
        if (ENV_MODE == ENV_DET_SMEM) {
            __syncthreads();
            for (int i = threadIdx.x; i < 3 * ne; i += SHADE_THREADS) {
                const uint64_t v = s_dwords[i];
                if (v) det_red_u64(a.det.words + (size_t)(i / ne) * a.det.n + (i % ne), v);
            }
            for (int i = threadIdx.x; i < nflag; i += SHADE_THREADS) { const uint32_t f = s_dflags[i]; if (f) atomicOr(a.det.flags + i, f); }
        }
    }
};

// dinc[3k + c] += dLg[c] * w[k]: the lane's 48 accumulators as 12 float4 in shared memory (acc4: the lane's first slot
// of [12][threads] 16-byte slots: conflict-free 128-bit accesses) — 12 LDS.128 + 48 FFMA + 12 STS.128 per sample
__device__ __forceinline__ void accumulate_dinc(float4* acc4, const float* dLg, const float* w) {
#pragma unroll
    for (int q = 0; q < 12; ++q) {
        float4 v = acc4[q * SHADE_THREADS];
        v.x = fmaf(dLg[(4 * q) % 3], w[(4 * q) / 3], v.x);
        v.y = fmaf(dLg[(4 * q + 1) % 3], w[(4 * q + 1) / 3], v.y);
        v.z = fmaf(dLg[(4 * q + 2) % 3], w[(4 * q + 2) / 3], v.z);
        v.w = fmaf(dLg[(4 * q + 3) % 3], w[(4 * q + 3) / 3], v.w);
        acc4[q * SHADE_THREADS] = v;
    }
}

template <typename K, typename... X>
static int shade_launch(K kernel, const ShadeArgs& a, int units, int num_sms, size_t smem, cudaStream_t stream, const X&... extra) {
    if (smem > 48 * 1024) R3DG_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, SHADE_THREADS, smem) != cudaSuccess || per_sm <= 0) per_sm = 2;
    const int want = (units + SHADE_WARPS - 1) / SHADE_WARPS;
    const int cap = num_sms * per_sm;                 // persistent CTAs: one env staging / flush per resident CTA
    const int grid = want < cap ? (want > 0 ? want : 1) : cap;
    kernel<<<grid, SHADE_THREADS, smem, stream>>>(a, extra...);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

static size_t inc_slot_bytes(int G, int var) { return var >= 1 ? (size_t)SHADE_WARPS * (32 / G) * SHADE_INC_STRIDE * sizeof(float) : 0; }

// texels of the texture the kernels read: the env, or every level of the filtered mode's pyramid
static size_t env_texels(const ShadeArgs& a, const EnvLevels& lv, bool filt) { return filt ? (size_t)lv.total : (size_t)a.He * a.We; }

template <int M> using EnvMode = std::integral_constant<int, M>;

// shading.cu, deterministic mode: the largest |cotangent| of the call's n cotangents of each kind into *a.det_scale
// (zeroed with the accumulators), and dL/denv from the accumulators
void launch_det_scale(const ShadeArgs& a, size_t n, int num_sms, cudaStream_t stream);
int launch_det_env(const ShadeArgs& a, cudaStream_t stream);

// Clears dL/denv (or the deterministic accumulators), picks the env-gradient mode from the texture size (nt texels),
// the deterministic flag and the highest mode allowed (`cap`), and calls run(EnvMode<mode>, args, env shared-memory
// bytes) unless P = 0; the deterministic mode first reduces the scale of the V views' cotangents and then converts its
// accumulators into dL/denv.
template <typename Run>
static int shade_backward(ShadeArgs a, int V, int cap, size_t nt, int num_sms, cudaStream_t stream, Run run) {
    if (a.det.words) {
        R3DG_CUDA_TRY(cudaMemsetAsync(a.det.words, 0, det_bytes(a.det.n) + sizeof(uint32_t), stream));   // + the scale word
        int rc = 0;
        if (a.P > 0) {
            launch_det_scale(a, (size_t)(V < 1 ? 1 : V) * a.P * 3, num_sms, stream);
            const size_t smem = EnvGrad<ENV_DET_SMEM>::smem_bytes(nt);     // larger textures use ENV_DET_GLOBAL
            a.env_in_smem = smem <= 64 * 1024;
            rc = a.env_in_smem ? run(EnvMode<ENV_DET_SMEM>(), a, smem) : run(EnvMode<ENV_DET_GLOBAL>(), a, 0);
        }
        if (rc) return rc;
        return launch_det_env(a, stream);
    }
    R3DG_CUDA_TRY(cudaMemsetAsync(a.d_env, 0, nt * 3 * sizeof(float), stream));
    if (a.P <= 0) return 0;
    // shared-memory cost of the env-gradient modes (kept within the 48 KB that need no opt-in on their own)
    const size_t tag_bytes = EnvGrad<ENV_TAG>::smem_bytes(nt), cas_bytes = EnvGrad<ENV_CAS>::smem_bytes(nt);
    if (cap >= ENV_TAG && tag_bytes <= 48 * 1024) { a.env_in_smem = 1; return run(EnvMode<ENV_TAG>(), a, tag_bytes); }
    if (cap >= ENV_CAS && cas_bytes <= 40 * 1024) { a.env_in_smem = 1; return run(EnvMode<ENV_CAS>(), a, cas_bytes); }
    a.env_in_smem = 0;
    return run(EnvMode<ENV_GLOBAL>(), a, 0);
}

}  // namespace r3dg
