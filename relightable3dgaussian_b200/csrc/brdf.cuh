// The shading step's per-Gaussian BRDF operands and GGX_specular (reference gaussian_renderer/neilf.py:374-406),
// forward and backward, shared by shading.cu (environment light) and lights.cu (point and directional lights).
// Both files are compiled with -fmad=false, so each op rounds as its PyTorch counterpart does.
#pragma once
#include "common.cuh"

namespace r3dg {

#define PI_F 3.14159274101257324f     // float32(np.pi)
#define INV_PI_F 0.318309873342514038f    // float32(1 / float32(np.pi))

struct GaussianOperands {
    float base[3], rough, n[3], Ns[3], V[3], vnorm, nx_raw[3];
    float a2, k;
    float inc[48];
};

// GGX_specular's forward quantities for one (Gaussian, direction, view); the shading step's sample record carries
// the same fields
struct GgxEval {
    float fs;
    float H[3], hn, NoL, NoV, NoH, VoH, NoL_r, NoV_r, NoH_r, VoH_r, p2, frac0, nom0, nom1, nom2, nom_r, nom;
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

// alpha^2 and k of the roughness o.rough
__device__ __forceinline__ void roughness_operands(GaussianOperands& o) {
    const float al = o.rough * o.rough;
    o.a2 = al * al;
    o.k = (al + 2.0f * o.rough + 1.0f) / 8.0f;
}

// the view-independent operands: material, raw normal, alpha^2 and k of the roughness (A: any argument record with
// the base_color [P,3], roughness [P] and normals [P,3] pointers)
template <class A>
__device__ __forceinline__ void load_material(const A& a, int g, GaussianOperands& o) {
#pragma unroll
    for (int c = 0; c < 3; ++c) { o.base[c] = a.base_color[3 * (size_t)g + c]; o.n[c] = a.normals[3 * (size_t)g + c]; }
    o.rough = a.roughness[g];
    roughness_operands(o);
}

// 1/x with one MUFU (<= 1 ulp), for the BACKWARD kernels only: their recomputed forward quantities and their gradient
// arithmetic tolerate a last-bit difference (tests: 1e-4 relative), while each of their IEEE divisions costs an
// FCHK and a slow-path branch.  The forward kernels keep the IEEE divisions of the PyTorch expression.
__device__ __forceinline__ float fast_rcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// GGX_specular (neilf.py:374-406) for the view V with the flipped normal Ns (o: alpha^2 and k)
// FAST: one-MUFU reciprocals (the backward kernels); the forward keeps IEEE divisions
template <bool FAST, class E>
__device__ __forceinline__ void eval_ggx(const float* V, const float* Ns, const GaussianOperands& o, float dx, float dy, float dz,
                                         E& e) {
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

// GGX_specular backward for the view V (flipped normal Ns) from dfs = dL/dfs: adds to drough and to dV = dL/dV.
// WANT_L: also writes dL = dL/dL_n, the gradient with respect to the NORMALISED light direction L_n (the shading
// step's directions carry no gradient; a point or directional light's do)
template <bool WANT_L = false, class E>
__device__ __forceinline__ void ggx_backward(const float* V, const float* Ns, const GaussianOperands& o, const E& e,
                                             float dfs, float& drough, float (&dV)[3], float* dL = nullptr) {
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
    float dNoL = 0.f;
    if (WANT_L) dNoL = (e.NoL_r >= 1e-6f && e.NoL_r <= 1.f) ? dnom2 * (1.0f - o.k) : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float dHraw = (dH[c] - e.H[c] * hdot) * ihn;
        dV[c] += dNoV * Ns[c] + dVoH * e.H[c] + 0.5f * dHraw;
        if (WANT_L) dL[c] = dNoL * Ns[c] + 0.5f * dHraw;
    }
}

}  // namespace r3dg
