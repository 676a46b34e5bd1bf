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
//    without atomics (see "environment-map gradient" below), summed and flushed once per CTA;
//  * the backward recomputes the forward per sample instead of saving [P,N,*] activations.
#include <algorithm>
#include <cstring>
#include <type_traits>
#include "common.cuh"
#include "detacc.cuh"
#include "kernels.h"

namespace r3dg {

#define SHADE_THREADS 128
#define SHADE_WARPS (SHADE_THREADS / 32)
#define PI_F 3.14159274101257324f     // float32(np.pi)

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

struct EnvTap { int idx[4]; float w[4]; };      // texel base offsets (float index of channel 0, or -1) + weights

// grid_sample(bilinear, zeros padding, align_corners=True) at the lat-long coordinates of dir d
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

struct GaussianOperands {
    float base[3], rough, n[3], Ns[3], V[3], vnorm, nx_raw[3];
    float a2, k;
    float inc[48];
};

// the view-dependent operands of one Gaussian: V = normalize(viewdir) (|viewdir| in vnorm) and the normal flipped
// towards the view, Ns = normalize(n) * sign(n . V)
__device__ __forceinline__ void view_operands(const float* n, const float* viewdir, float* V, float& vnorm, float* Ns) {
    const float v0 = viewdir[0], v1 = viewdir[1], v2 = viewdir[2];
    vnorm = fmaxf(sqrtf(v0 * v0 + v1 * v1 + v2 * v2), 1e-12f);             // F.normalize eps
    V[0] = v0 / vnorm; V[1] = v1 / vnorm; V[2] = v2 / vnorm;
    const float nn = fmaxf(sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]), 1e-12f);
    const float N0 = n[0] / nn, N1 = n[1] / nn, N2 = n[2] / nn;
    const float nov = V[0] * N0 + V[1] * N1 + V[2] * N2;
    const float sg = nov > 0.f ? 1.f : (nov < 0.f ? -1.f : 0.f);             // torch.sign
    Ns[0] = N0 * sg; Ns[1] = N1 * sg; Ns[2] = N2 * sg;
}

// the view-independent operands: material, raw normal, alpha^2 and k of the roughness
__device__ __forceinline__ void load_material(const ShadeArgs& a, int g, GaussianOperands& o) {
#pragma unroll
    for (int c = 0; c < 3; ++c) { o.base[c] = a.base_color[3 * (size_t)g + c]; o.n[c] = a.normals[3 * (size_t)g + c]; }
    o.rough = a.roughness[g];
    const float al = o.rough * o.rough;
    o.a2 = al * al;
    o.k = (al + 2.0f * o.rough + 1.0f) / 8.0f;
}

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
#define SHADE_INC_STRIDE 52       // floats per group slot: 16-byte aligned, bank-staggered (52 mod 32 = 20)

template <int G>
__device__ __forceinline__ void stage_incidents(const ShadeArgs& a, int g, float* slot, int sub) {
    const float4* src = reinterpret_cast<const float4*>(a.incidents + 48 * (size_t)g);
    float4* dst = reinterpret_cast<float4*>(slot);
    for (int q = sub; q < 12; q += G) dst[q] = src[q];
    __syncwarp();
}

// 1/x with one MUFU (<= 1 ulp), for the BACKWARD kernel only: its recomputed forward quantities and its gradient
// arithmetic tolerate a last-bit difference (tests: 1e-4 relative), while each of its IEEE divisions per sample costs an
// FCHK and a slow-path branch.  The forward kernel keeps the
// IEEE divisions of the PyTorch expression.
__device__ __forceinline__ float fast_rcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
#define INV_PI_F 0.318309873342514038f    // float32(1 / float32(np.pi))

struct SampleEval {       // forward quantities of one (Gaussian, direction) pair
    float local_raw[3], glob[3], ndi, fs;
    float w[16];
    EnvTap taps;
    // GGX intermediates for the backward
    float H[3], hn, NoL, NoV, NoH, VoH, NoL_r, NoV_r, NoH_r, VoH_r, p2, frac0, nom0, nom1, nom2, nom_r, nom;
};

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

// the local SH light (before its clamp) and n.w with the raw normal
template <bool INC_SMEM>
__device__ __forceinline__ void eval_local(const GaussianOperands& o, const float* __restrict__ sinc, float dx, float dy, float dz,
                                           SampleEval& e) {
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

// GGX_specular (neilf.py:374-406) for the view V with the flipped normal Ns (o: alpha^2 and k)
// FAST: one-MUFU reciprocals (the backward kernels); the forward keeps IEEE divisions
template <bool FAST>
__device__ __forceinline__ void eval_ggx(const float* V, const float* Ns, const GaussianOperands& o, float dx, float dy, float dz,
                                         SampleEval& e) {
    const float ln = fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-12f);
    float L0, L1, L2;
    if (FAST) { const float il = fast_rcp(ln); L0 = dx * il; L1 = dy * il; L2 = dz * il; }
    else { L0 = dx / ln; L1 = dy / ln; L2 = dz / ln; }
    const float h0 = (L0 + V[0]) / 2.0f, h1 = (L1 + V[1]) / 2.0f, h2 = (L2 + V[2]) / 2.0f;
    e.hn = fmaxf(sqrtf(h0 * h0 + h1 * h1 + h2 * h2), 1e-12f);
    if (FAST) { const float ih = fast_rcp(e.hn); e.H[0] = h0 * ih; e.H[1] = h1 * ih; e.H[2] = h2 * ih; }
    else { e.H[0] = h0 / e.hn; e.H[1] = h1 / e.hn; e.H[2] = h2 / e.hn; }
    e.NoL_r = Ns[0] * L0 + Ns[1] * L1 + Ns[2] * L2;
    e.NoV_r = Ns[0] * V[0] + Ns[1] * V[1] + Ns[2] * V[2];
    e.NoH_r = Ns[0] * e.H[0] + Ns[1] * e.H[1] + Ns[2] * e.H[2];
    e.VoH_r = V[0] * e.H[0] + V[1] * e.H[1] + V[2] * e.H[2];
    e.NoL = fminf(fmaxf(e.NoL_r, 1e-6f), 1.f); e.NoV = fminf(fmaxf(e.NoV_r, 1e-6f), 1.f);
    e.NoH = fminf(fmaxf(e.NoH_r, 1e-6f), 1.f); e.VoH = fminf(fmaxf(e.VoH_r, 1e-6f), 1.f);
    const float FMi = (-5.55473f * e.VoH - 6.98316f) * e.VoH;
    e.p2 = exp2f(FMi);
    e.frac0 = 0.04f + (1.0f - 0.04f) * e.p2;
    e.nom0 = e.NoH * e.NoH * (o.a2 - 1.0f) + 1.0f;
    e.nom1 = e.NoV * (1.0f - o.k) + o.k;
    e.nom2 = e.NoL * (1.0f - o.k) + o.k;
    e.nom_r = 4.0f * PI_F * e.nom0 * e.nom0 * e.nom1 * e.nom2;
    e.nom = fminf(fmaxf(e.nom_r, 1e-6f), 4.0f * PI_F);
    e.fs = FAST ? e.frac0 * o.a2 * fast_rcp(e.nom) : e.frac0 * o.a2 / e.nom;
}

template <bool SMEM_ENV, bool INC_SMEM, bool FAST = false>
__device__ __forceinline__ void eval_sample(const ShadeArgs& a, const GaussianOperands& o, const float* __restrict__ env,
                                            const float* __restrict__ sinc, float dx, float dy, float dz, float vis, SampleEval& e) {
    eval_env<SMEM_ENV>(a.transform, env, a.He, a.We, dx, dy, dz, vis, e);
    eval_local<INC_SMEM>(o, sinc, dx, dy, dz, e);
    eval_ggx<FAST>(o.V, o.Ns, o, dx, dy, dz, e);
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

template <bool SMEM_ENV, int G, int VAR>
__global__ void __launch_bounds__(SHADE_THREADS, VAR == 1 ? 6 : 1) shade_fwd_kernel(const ShadeArgs a) {
    extern __shared__ __align__(16) float s_fwd[];     // [incident slots (VAR 1)][env texture (SMEM_ENV)]
    constexpr int GPW = 32 / G;                    // Gaussians per warp
    constexpr int INC_FLOATS = VAR >= 1 ? SHADE_WARPS * GPW * SHADE_INC_STRIDE : 0;
    float* s_env = s_fwd + INC_FLOATS;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & (G - 1), grp = lane / G;
    float* sinc = s_fwd + (warp * GPW + grp) * SHADE_INC_STRIDE;
    if (SMEM_ENV) {
        for (int i = threadIdx.x; i < a.He * a.We * 3; i += SHADE_THREADS) s_env[i] = a.env[i];
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
            SampleEval e;
            eval_sample<SMEM_ENV, (VAR >= 1)>(a, o, env, sinc, dx, dy, dz, vis, e);
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

    // bytes of `s_mem` the constructor lays out for an He x We texture (0 for the global-memory modes):
    // ENV_CAS: [env ne][grad ne]; ENV_TAG: [env ne (padded to 4)][per warp: float4 grad[nt]][per warp: tag[nt] padded to 16];
    // ENV_DET_SMEM: [env ne (padded to 2)][accumulator words 3 ne][flag words (ne + 15) / 16]
    static __host__ __device__ size_t smem_bytes(int He, int We) {
        const size_t nt = (size_t)He * We, ne = nt * 3;
        if (ENV_MODE == ENV_CAS) return 2 * ne * sizeof(float);
        if (ENV_MODE == ENV_TAG) return ((ne + 3) & ~(size_t)3) * sizeof(float) + SHADE_WARPS * (nt * sizeof(float4) + ((nt + 15) & ~(size_t)15));
        if (ENV_MODE == ENV_DET_SMEM) return ((ne + 1) & ~(size_t)1) * sizeof(float) + 3 * ne * sizeof(uint64_t) + (ne + 15) / 16 * sizeof(uint32_t);
        return 0;
    }

    __device__ __forceinline__ EnvGrad(const ShadeArgs& a, float* s_mem, int warp) {
        nt = a.He * a.We; ne = nt * 3;
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
    __device__ __forceinline__ void scatter(const ShadeArgs& a, const EnvTap& taps, const float* dG, int lane) {
        if (ENV_MODE == ENV_TAG) {
            const bool any = dG[0] != 0.f || dG[1] != 0.f || dG[2] != 0.f;
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int texel = (any && taps.idx[t] >= 0) ? taps.idx[t] / 3 : -1;
                warp_private_add(wgrad, wtag, texel, dG[0] * taps.w[t], dG[1] * taps.w[t], dG[2] * taps.w[t], lane);
            }
        } else if (ENV_MODE == ENV_DET_SMEM || ENV_MODE == ENV_DET_GLOBAL) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                if (dG[c] != 0.f) {
#pragma unroll
                    for (int t = 0; t < 4; ++t)
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
                    for (int t = 0; t < 4; ++t) if (taps.idx[t] >= 0) atomicAdd(genv + taps.idx[t] + c, dG[c] * taps.w[t]);
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

// GGX_specular backward for the view V (flipped normal Ns) from dfs = dL/dfs: adds to drough and to dV = dL/dV
__device__ __forceinline__ void ggx_backward(const float* V, const float* Ns, const GaussianOperands& o, const SampleEval& e,
                                             float dfs, float& drough, float (&dV)[3]) {
    const float inom = fast_rcp(e.nom);
    const float dfrac = dfs * inom;
    const float dnom = -dfs * (e.frac0 * o.a2) * inom * inom;
    const float dnom_r = (e.nom_r >= 1e-6f && e.nom_r <= 4.0f * PI_F) ? dnom : 0.f;
    const float dnom0 = dnom_r * 8.0f * PI_F * e.nom0 * e.nom1 * e.nom2;
    const float dnom1 = dnom_r * 4.0f * PI_F * e.nom0 * e.nom0 * e.nom2;
    const float dnom2 = dnom_r * 4.0f * PI_F * e.nom0 * e.nom0 * e.nom1;
    const float dfrac0 = dfrac * o.a2;
    const float da2 = dfrac * e.frac0 + dnom0 * e.NoH * e.NoH;
    const float dk = dnom1 * (1.0f - e.NoV) + dnom2 * (1.0f - e.NoL);
    const float r = o.rough;
    drough += da2 * 4.0f * r * r * r + dk * (2.0f * r + 2.0f) / 8.0f;
    const float dNoH = (e.NoH_r >= 1e-6f && e.NoH_r <= 1.f) ? dnom0 * 2.0f * e.NoH * (o.a2 - 1.0f) : 0.f;
    const float dNoV = (e.NoV_r >= 1e-6f && e.NoV_r <= 1.f) ? dnom1 * (1.0f - o.k) : 0.f;
    const float dVoH = (e.VoH_r >= 1e-6f && e.VoH_r <= 1.f)
                           ? dfrac0 * (1.0f - 0.04f) * e.p2 * 0.693147180559945f * (2.0f * -5.55473f * e.VoH - 6.98316f) : 0.f;
    float dH[3], hdot = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) { dH[c] = dNoH * Ns[c] + dVoH * V[c]; hdot += e.H[c] * dH[c]; }
    const float ihn = fast_rcp(e.hn);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float dHraw = (dH[c] - e.H[c] * hdot) * ihn;
        dV[c] += dNoV * Ns[c] + dVoH * e.H[c] + 0.5f * dHraw;
    }
}

// resident CTAs the register allocation is pinned to: variant 1 -> 3 (<= 168 registers); variant 2 ->
// 3 with the warp-private env copies (67 KB of shared memory per CTA) or the deterministic modes (their fixed-point
// conversion spills at 102 registers), 5 otherwise (<= 102 registers)
template <int ENV_MODE, int G, int VAR>
__global__ void __launch_bounds__(SHADE_THREADS, VAR == 0 ? 1 : VAR == 1 ? 3 : (ENV_MODE <= 1 ? 5 : 3)) shade_bwd_kernel(const ShadeArgs a) {
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
    EnvGrad<ENV_MODE> eg(a, s_mem, warp);
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
            SampleEval e;
            eval_sample<SMEM_ENV, (VAR >= 1), true>(a, o, eg.env, sinc, dx, dy, dz, vis, e);
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

template <bool SMEM_ENV>
__global__ void __launch_bounds__(SHADE_THREADS, 3) shade_views_fwd_kernel(const ShadeArgs a, const ViewChunk vc) {
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
        for (int i = threadIdx.x; i < a.He * a.We * 3; i += SHADE_THREADS) s_env[i] = a.env[i];
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
            SampleEval e;
            if (!pvt) eval_env<SMEM_ENV>(a.transform, env, a.He, a.We, dx, dy, dz, vis, e);
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
                if (pvt) eval_env<SMEM_ENV>(a.transform + 9 * (size_t)(vc.v0 + v), env, a.He, a.We, dx, dy, dz, vis, e);
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
template <int ENV_MODE>
__global__ void __launch_bounds__(SHADE_THREADS, 3) shade_views_bwd_kernel(const ShadeArgs a, const ViewChunk vc) {
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
    EnvGrad<ENV_MODE> eg(a, s_vbwd + INC_FLOATS + DINC_FLOATS + SLOT_FLOATS + DV_FLOATS, warp);
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
            SampleEval e;
            eval_env<SMEM_ENV>(a.transform, eg.env, a.He, a.We, dx, dy, dz, vis, e);
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

template <bool SMEM>
static int launch_fwd(const ShadeArgs& a, int num_sms, size_t env_smem, cudaStream_t stream) {
    const int G = knob(0);
    const int var = G == 8 ? knob(2) : 0;              // the shared-memory variants are built for the default group width
    const size_t smem = env_smem + inc_slot_bytes(G, var);
    const int units = (a.P + 32 / G - 1) / (32 / G);
    if (G == 8) return var ? shade_launch(shade_fwd_kernel<SMEM, 8, 1>, a, units, num_sms, smem, stream)
                           : shade_launch(shade_fwd_kernel<SMEM, 8, 0>, a, units, num_sms, smem, stream);
    if (G == 16) return shade_launch(shade_fwd_kernel<SMEM, 16, 0>, a, units, num_sms, smem, stream);
    return shade_launch(shade_fwd_kernel<SMEM, 32, 0>, a, units, num_sms, smem, stream);
}

int launch_shade_forward(ShadeArgs a, int num_sms, cudaStream_t stream) {
    if (a.P <= 0) return 0;
    const size_t env_bytes = (size_t)a.He * a.We * 3 * sizeof(float);
    const bool smem = env_bytes <= 40 * 1024;
    a.env_in_smem = smem;
    return smem ? launch_fwd<true>(a, num_sms, env_bytes, stream) : launch_fwd<false>(a, num_sms, 0, stream);
}

template <int MODE>
static int launch_bwd(const ShadeArgs& a, int num_sms, size_t env_smem, cudaStream_t stream) {
    const int G = knob(0);
    const int var = G == 8 ? knob(3) : 0;
    const size_t smem = env_smem + inc_slot_bytes(G, var) + (var == 2 ? (size_t)48 * SHADE_THREADS * sizeof(float) : 0);
    const int units = (a.P + 32 / G - 1) / (32 / G);
    if (G == 8) return var == 2 ? shade_launch(shade_bwd_kernel<MODE, 8, 2>, a, units, num_sms, smem, stream)
                     : var == 1 ? shade_launch(shade_bwd_kernel<MODE, 8, 1>, a, units, num_sms, smem, stream)
                                : shade_launch(shade_bwd_kernel<MODE, 8, 0>, a, units, num_sms, smem, stream);
    if (G == 16) return shade_launch(shade_bwd_kernel<MODE, 16, 0>, a, units, num_sms, smem, stream);
    return shade_launch(shade_bwd_kernel<MODE, 32, 0>, a, units, num_sms, smem, stream);
}

template <int M> using EnvMode = std::integral_constant<int, M>;

// Clears dL/denv (or the deterministic accumulators), picks the env-gradient mode from the texture size, the deterministic
// flag and the highest mode allowed (`cap`), and calls run(EnvMode<mode>, args, env shared-memory bytes) unless P = 0;
// the deterministic mode first reduces the scale of the V views' cotangents and then converts its accumulators into
// dL/denv.
template <typename Run>
static int shade_backward(ShadeArgs a, int V, int cap, int num_sms, cudaStream_t stream, Run run) {
    if (a.det.words) {
        R3DG_CUDA_TRY(cudaMemsetAsync(a.det.words, 0, det_bytes(a.det.n) + sizeof(uint32_t), stream));   // + the scale word
        int rc = 0;
        if (a.P > 0) {
            const size_t n = (size_t)(V < 1 ? 1 : V) * a.P * 3;
            const unsigned blocks = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)4 * num_sms);
            det_scale_kernel<<<blocks, 256, 0, stream>>>(n, a.g_pbr, a.g_diffuse, a.g_specular, a.det_scale);
            const size_t smem = EnvGrad<ENV_DET_SMEM>::smem_bytes(a.He, a.We);     // larger textures use ENV_DET_GLOBAL
            a.env_in_smem = smem <= 64 * 1024;
            rc = a.env_in_smem ? run(EnvMode<ENV_DET_SMEM>(), a, smem) : run(EnvMode<ENV_DET_GLOBAL>(), a, 0);
        }
        if (rc) return rc;
        det_env_kernel<<<(unsigned)((a.det.n + 255) / 256), 256, 0, stream>>>(a.det, a.det_scale, a.d_env);
        R3DG_CUDA_TRY(cudaGetLastError());
        return 0;
    }
    R3DG_CUDA_TRY(cudaMemsetAsync(a.d_env, 0, (size_t)a.He * a.We * 3 * sizeof(float), stream));
    if (a.P <= 0) return 0;
    // shared-memory cost of the env-gradient modes (kept within the 48 KB that need no opt-in on their own)
    const size_t tag_bytes = EnvGrad<ENV_TAG>::smem_bytes(a.He, a.We), cas_bytes = EnvGrad<ENV_CAS>::smem_bytes(a.He, a.We);
    if (cap >= ENV_TAG && tag_bytes <= 48 * 1024) { a.env_in_smem = 1; return run(EnvMode<ENV_TAG>(), a, tag_bytes); }
    if (cap >= ENV_CAS && cas_bytes <= 40 * 1024) { a.env_in_smem = 1; return run(EnvMode<ENV_CAS>(), a, cas_bytes); }
    a.env_in_smem = 0;
    return run(EnvMode<ENV_GLOBAL>(), a, 0);
}

int launch_shade_backward(ShadeArgs a, int num_sms, cudaStream_t stream) {
    return shade_backward(a, 1, knob(1), num_sms, stream, [&](auto mode, const ShadeArgs& x, size_t env_smem) {
        return launch_bwd<decltype(mode)::value>(x, num_sms, env_smem, stream);
    });
}

// ---- several views: one launch per SHADE_VIEW_CHUNK views ------------------------------------------
static size_t view_slot_bytes(int slot_floats) { return (size_t)SHADE_WARPS * 4 * SHADE_VIEW_CHUNK * slot_floats * sizeof(float); }

int launch_shade_views_forward(ShadeArgs a, int V, int per_view_transform, int num_sms, cudaStream_t stream) {
    if (a.P <= 0) return 0;
    const size_t env_bytes = (size_t)a.He * a.We * 3 * sizeof(float);
    const bool smem_env = env_bytes <= 40 * 1024;     // as the one-view forward
    a.env_in_smem = smem_env;
    const int K = view_fwd_sums(per_view_transform && a.mean_lights);
    const size_t smem = inc_slot_bytes(8, 1) + view_slot_bytes(VIEW_FWD_SLOT) + (size_t)K * SHADE_VIEW_CHUNK * SHADE_THREADS * sizeof(float) +
                        (smem_env ? env_bytes : 0);
    const int units = (a.P + 3) / 4;
    for (int v0 = 0; v0 < V; v0 += SHADE_VIEW_CHUNK) {
        const ViewChunk vc{v0, V - v0 < SHADE_VIEW_CHUNK ? V - v0 : SHADE_VIEW_CHUNK, per_view_transform, 0};
        const int rc = smem_env ? shade_launch(shade_views_fwd_kernel<true>, a, units, num_sms, smem, stream, vc)
                                : shade_launch(shade_views_fwd_kernel<false>, a, units, num_sms, smem, stream, vc);
        if (rc) return rc;
    }
    return 0;
}

// the env-gradient mode as the one-view backward picks it at its default highest mode (the view kernels have no knobs)
int launch_shade_views_backward(ShadeArgs a, int V, int num_sms, cudaStream_t stream) {
    return shade_backward(a, V, ENV_CAS, num_sms, stream, [&](auto mode, const ShadeArgs& x, size_t env_smem) {
        constexpr int M = decltype(mode)::value;
        if constexpr (M == ENV_TAG) return (int)R3DG_ERR_UNSUPPORTED;     // above the cap: never selected
        else {
            const size_t smem = inc_slot_bytes(8, 2) + (size_t)48 * SHADE_THREADS * sizeof(float) + view_slot_bytes(VIEW_BWD_SLOT) +
                                (size_t)3 * SHADE_VIEW_CHUNK * SHADE_THREADS * sizeof(float) + env_smem;
            for (int v0 = 0; v0 < V; v0 += SHADE_VIEW_CHUNK) {
                const ViewChunk vc{v0, V - v0 < SHADE_VIEW_CHUNK ? V - v0 : SHADE_VIEW_CHUNK, 0, v0 > 0};
                const int rc = shade_launch(shade_views_bwd_kernel<M>, x, (x.P + 3) / 4, num_sms, smem, stream, vc);
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

int r3dg_render_equation_forward(const r3dg_shade_args* s, r3dg_stream_t stream) {
    ShadeArgs a;
    int rc = fill_args(s, a);
    if (rc) return rc;
    if (a.P > 0 && (!a.pbr || !a.diffuse || !a.specular)) return R3DG_ERR_BAD_ARG;
    if ((a.mean_lights != nullptr) != (a.mean_local != nullptr) || (a.mean_lights != nullptr) != (a.mean_global != nullptr)) return R3DG_ERR_BAD_ARG;
    if ((a.s_lights != nullptr) != (a.s_local != nullptr) || (a.s_lights != nullptr) != (a.s_global != nullptr)) return R3DG_ERR_BAD_ARG;
    if (s->V > 1) {
        if (a.s_lights) return R3DG_ERR_UNSUPPORTED;               // no per-sample [V,P,N,3] outputs
        if (a.mean_lights && !a.mean_vis) return R3DG_ERR_BAD_ARG;
        return launch_shade_views_forward(a, s->V, s->transform_per_view && a.transform, num_sms(), (cudaStream_t)stream);
    }
    return launch_shade_forward(a, num_sms(), (cudaStream_t)stream);
}

int r3dg_render_equation_backward(const r3dg_shade_args* s, r3dg_stream_t stream) {
    ShadeArgs a;
    int rc = fill_args(s, a);
    if (rc) return rc;
    if (!a.g_pbr || !a.d_base || !a.d_rough || !a.d_view || !a.d_incidents || !a.d_env) return R3DG_ERR_BAD_ARG;
    if (s->V > 1 && s->transform_per_view && a.transform) return R3DG_ERR_UNSUPPORTED;    // forward only
    if (s->deterministic) {
        const size_t n = (size_t)a.He * a.We * 3;
        if (!s->det_work || s->det_work_bytes < r3dg_shade_det_bytes(a.He, a.We)) return R3DG_ERR_BAD_ARG;
        a.det = det_acc(s->det_work, n);
        a.det_scale = (uint32_t*)((char*)s->det_work + det_bytes(n));
    }
    return s->V > 1 ? launch_shade_views_backward(a, s->V, num_sms(), (cudaStream_t)stream)
                    : launch_shade_backward(a, num_sms(), (cudaStream_t)stream);
}

// the accumulators and the call's scale word
size_t r3dg_shade_det_bytes(int env_h, int env_w) {
    return env_h > 0 && env_w > 0 ? det_bytes((size_t)env_h * env_w * 3) + 256 : 0;
}

}  // extern "C"
