// The importance sampler of the environment light (include/r3dg_b200.h, IMPORTANCE SAMPLING; DESIGN.md §4.31): the
// env table's layout, the three strategies (env, GGX, cosine), their pdfs and the balance-heuristic area of a sample.
// A sample's direction and area must be the same bits wherever they are computed, whatever the file's contraction
// setting, so every operation is rounded on its own with explicit intrinsics (as fib_sample and rotate_from_z are).
#pragma once
#include "bvh.cuh"
#include "lights.cuh"

namespace r3dg {

#define IS_PI 3.14159274101257324f          // float32(pi)
#define IS_TWO_PI 6.28318548202514648f      // float32(2 pi)

// The table of r3dg_env_sampler_build, in floats: a header {He, We (int32 bits), 0, 0}, the build's fp64 row weights
// [He] (two floats each), the row CDF [He+1], 1 - cos and 1 + cos of the row bands' edges [He+1] each (accurate near
// either pole, where cos itself cannot resolve a direction in fp32), the column CDFs [He][We] (We - 1 cells per row;
// entry We - 1 is 1) and the cell pdfs [He][We-1] (per steradian).
__host__ __device__ inline size_t env_sampler_floats(int He, int We) {
    return 4 + 2 * (size_t)He + 3 * ((size_t)He + 1) + (size_t)He * We + (size_t)He * (We - 1);
}

struct EnvTable {
    int He, We;
    const float *row_cdf, *vers, *covers, *col_cdf, *pdf;
    float dphi;                                      // 2 pi / (We - 1), rounded once
    EnvTable() = default;
    __device__ __forceinline__ explicit EnvTable(const float* t) {
        He = __float_as_int(t[0]); We = __float_as_int(t[1]);
        row_cdf = t + 4 + 2 * (size_t)He;
        vers = row_cdf + He + 1;
        covers = vers + He + 1;
        col_cdf = covers + He + 1;
        pdf = col_cdf + (size_t)He * We;
        dphi = div_(IS_TWO_PI, (float)(We - 1));
    }
};

// the largest k in [0, n) with c[k] <= u (c ascending, c[0] <= u)
__device__ __forceinline__ int cdf_find(const float* c, int n, float u) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (c[mid] <= u) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// The two numbers of sample k of a strategy with n samples: a rank-1 lattice rotated by the hash h (integer arithmetic,
// then the top 24 bits, exact in fp32)
__device__ __forceinline__ uint32_t is_hash(uint32_t seed, uint32_t q, uint32_t s) { return rect_hash(seed, q, s); }
__device__ __forceinline__ void lattice_uv(uint32_t h, int k, int n, float& u1, float& u2) {
    const uint32_t h1 = lowbias32(h ^ 0u), h2 = lowbias32(h ^ 1u);
    const uint32_t a = (uint32_t)(((unsigned long long)k << 32) / (unsigned long long)n) + h1;
    const uint32_t b = (uint32_t)k * 0x9E3779B9u + h2;
    u1 = hash_unit(a); u2 = hash_unit(b);
}

__device__ __forceinline__ float dot3r(float ax, float ay, float az, float bx, float by, float bz) {
    return add_(add_(mul_(ax, bx), mul_(ay, by)), mul_(az, bz));
}
__device__ __forceinline__ float3 normalize_r(float x, float y, float z) { return unit_normal(x, y, z); }

// env space d_e = T d (T: the EnvLight transform, row-major, or NULL) and world space d = T^T d_e
__device__ __forceinline__ float3 to_env(const float* T, float3 d) {
    if (!T) return d;
    return make_float3(dot3r(T[0], T[1], T[2], d.x, d.y, d.z), dot3r(T[3], T[4], T[5], d.x, d.y, d.z),
                       dot3r(T[6], T[7], T[8], d.x, d.y, d.z));
}
__device__ __forceinline__ float3 from_env(const float* T, float3 e) {
    if (!T) return e;
    return normalize_r(dot3r(T[0], T[3], T[6], e.x, e.y, e.z), dot3r(T[1], T[4], T[7], e.x, e.y, e.z),
                       dot3r(T[2], T[5], T[8], e.x, e.y, e.z));
}

// ---- env strategy: row by the row CDF, column by the row's column CDF, uniform in solid angle inside the cell ----
__device__ __forceinline__ float3 env_sample(const EnvTable& t, const float* T, float u1, float u2) {
    const int j = cdf_find(t.row_cdf, t.He, u1);
    const float t1 = div_(sub_(u1, t.row_cdf[j]), sub_(t.row_cdf[j + 1], t.row_cdf[j]));
    const float* cc = t.col_cdf + (size_t)j * t.We;
    const int i = cdf_find(cc, t.We - 1, u2);
    const float t2 = div_(sub_(u2, cc[i]), sub_(cc[i + 1], cc[i]));
    // cos theta = cos lo + t1 (cos hi - cos lo), formed as 1 - v (northern rows) or w - 1 (southern rows)
    float cz, sz;
    if (2 * j <= t.He - 1) {
        const float v = add_(t.vers[j], mul_(t1, sub_(t.vers[j + 1], t.vers[j])));
        cz = sub_(1.0f, v); sz = sqrt_(fmaxf(mul_(v, sub_(2.0f, v)), 0.0f));
    } else {
        const float w = add_(t.covers[j], mul_(t1, sub_(t.covers[j + 1], t.covers[j])));
        cz = sub_(w, 1.0f); sz = sqrt_(fmaxf(mul_(w, sub_(2.0f, w)), 0.0f));
    }
    const float az = sub_(IS_PI, mul_(add_((float)i - 0.5f, t2), t.dphi));    // the lookup's column i - 1/2 + t2
    return from_env(T, make_float3(mul_(sz, cosf(az)), mul_(sz, sinf(az)), cz));
}
// its pdf per steradian at the world direction d: the pdf of the cell d falls in
__device__ __forceinline__ float env_pdf(const EnvTable& t, const float* T, float3 d) {
    const float3 e = to_env(T, d);
    const int lo = cdf_find(t.vers, t.He, sub_(1.0f, e.z));          // row j: vers[j] <= 1 - z < vers[j+1]
    int i = (int)floorf(add_(div_(sub_(IS_PI, atan2f(e.y, e.x)), t.dphi), 0.5f));
    if (i >= t.We - 1) i -= t.We - 1;
    if (i < 0) i = 0;
    return t.pdf[(size_t)lo * (t.We - 1) + i];
}

// ---- GGX strategy: the NDF of alpha^2 = max(r^4, 1e-7) around Ns (the normal flipped towards V), reflected about h ----
struct GgxFrame {
    float V[3], Ns[3], a2;
    bool lobe;                                       // false when n.V = 0: Ns = 0, no GGX lobe to sample
};
__device__ __forceinline__ GgxFrame ggx_frame(float3 nh, float vx, float vy, float vz, float rough) {
    GgxFrame f;
    const float3 v = normalize_r(vx, vy, vz);
    f.V[0] = v.x; f.V[1] = v.y; f.V[2] = v.z;
    const float nov = dot3r(nh.x, nh.y, nh.z, v.x, v.y, v.z);
    const float sg = nov > 0.f ? 1.f : (nov < 0.f ? -1.f : 0.f);
    f.Ns[0] = mul_(nh.x, sg); f.Ns[1] = mul_(nh.y, sg); f.Ns[2] = mul_(nh.z, sg);
    const float r2 = mul_(rough, rough);
    f.a2 = fmaxf(mul_(r2, r2), 1e-7f);
    f.lobe = sg != 0.f;
    return f;
}
// the direction of (u1, u2); `ok` is false when its half-vector faces away from V, or when there is no lobe (neither
// is a sample of ggx_pdf: area 0)
__device__ __forceinline__ float3 ggx_sample(const GgxFrame& f, float u1, float u2, bool& ok) {
    // cos^2 = (1 - u1) / den and sin^2 = a2 u1 / den: no cancellation at a small alpha
    const float den = add_(1.0f, mul_(sub_(f.a2, 1.0f), u1));
    const float ch = sqrt_(div_(sub_(1.0f, u1), den)), sh = sqrt_(div_(mul_(f.a2, u1), den));
    const float ph = mul_(IS_TWO_PI, u2);
    const float3 h = rotate_from_z(f.Ns[0], f.Ns[1], f.Ns[2], make_float3(mul_(sh, cosf(ph)), mul_(sh, sinf(ph)), ch));
    const float vh = dot3r(f.V[0], f.V[1], f.V[2], h.x, h.y, h.z);
    ok = f.lobe && vh > 0.f;
    const float w = mul_(2.0f, vh);
    return normalize_r(sub_(mul_(w, h.x), f.V[0]), sub_(mul_(w, h.y), f.V[1]), sub_(mul_(w, h.z), f.V[2]));
}
// D(h) (Ns.h) / (4 V.h) with h = normalize(V + l); 0 when Ns.h <= 0 or V.h <= 0.  D's denominator
// (Ns.h)^2 (a2 - 1) + 1 is formed as |Ns x h|^2 + a2 (Ns.h)^2: near the lobe's peak 1 - (Ns.h)^2 would cancel to about
// a2 and amplify the rounding of Ns.h by 1 / a2
__device__ __forceinline__ float ggx_pdf(const GgxFrame& f, float3 l) {
    const float3 h = normalize_r(add_(f.V[0], l.x), add_(f.V[1], l.y), add_(f.V[2], l.z));
    const float nh = dot3r(f.Ns[0], f.Ns[1], f.Ns[2], h.x, h.y, h.z);
    const float vh = dot3r(f.V[0], f.V[1], f.V[2], h.x, h.y, h.z);
    if (!(nh > 0.f) || !(vh > 0.f)) return 0.f;
    const float cx = sub_(mul_(f.Ns[1], h.z), mul_(f.Ns[2], h.y)), cy = sub_(mul_(f.Ns[2], h.x), mul_(f.Ns[0], h.z)),
                cz = sub_(mul_(f.Ns[0], h.y), mul_(f.Ns[1], h.x));
    const float den = add_(dot3r(cx, cy, cz, cx, cy, cz), mul_(f.a2, mul_(nh, nh)));
    const float D = div_(f.a2, mul_(IS_PI, mul_(den, den)));
    return div_(mul_(D, nh), mul_(4.0f, vh));
}

// ---- cosine strategy around the unit normal ----
__device__ __forceinline__ float3 cos_sample(float3 nh, float u1, float u2) {
    const float r = sqrt_(u1), ph = mul_(IS_TWO_PI, u2);
    return rotate_from_z(nh.x, nh.y, nh.z, make_float3(mul_(r, cosf(ph)), mul_(r, sinf(ph)), sqrt_(sub_(1.0f, u1))));
}
__device__ __forceinline__ float cos_pdf(float3 nh, float3 d) {
    return div_(fmaxf(dot3r(nh.x, nh.y, nh.z, d.x, d.y, d.z), 0.f), IS_PI);
}

// The sampler of one shading point: N = n_env + n_ggx + n_cos samples in that order, the row (or pixel) index q.
struct ImportanceSampler {
    EnvTable t;                                      // the table's views, made on the device from `table`
    const float* table;                              // r3dg_env_sampler_build's output, or NULL: no sampler
    const float* T;
    int N, n_env, n_ggx;
    uint32_t seed;
};

// Sample i of shading point q (unit normal nh; GGX frame f, read only when n_ggx > 0): its direction, and its area
// N / (n_env p_env + n_ggx p_ggx + n_cos p_cos), 0 when that denominator is not a positive finite number
__device__ __forceinline__ float3 importance_sample(const ImportanceSampler& s, uint32_t q, int i, float3 nh, const GgxFrame& f,
                                                    float& area) {
    const int n_eg = s.n_env + s.n_ggx, n_cos = s.N - n_eg;
    const int strat = i < s.n_env ? 0 : (i < n_eg ? 1 : 2);
    const int k = strat == 0 ? i : (strat == 1 ? i - s.n_env : i - n_eg);
    const int ns = strat == 0 ? s.n_env : (strat == 1 ? s.n_ggx : n_cos);
    float u1, u2;
    lattice_uv(is_hash(s.seed, q, (uint32_t)strat), k, ns, u1, u2);
    bool ok = true;
    const float3 d = strat == 0 ? env_sample(s.t, s.T, u1, u2) : (strat == 1 ? ggx_sample(f, u1, u2, ok) : cos_sample(nh, u1, u2));
    float den = 0.f;                                  // ((n_env p_env + n_ggx p_ggx) + n_cos p_cos)
    if (s.n_env > 0) den = mul_((float)s.n_env, env_pdf(s.t, s.T, d));
    if (s.n_ggx > 0) den = add_(den, mul_((float)s.n_ggx, ggx_pdf(f, d)));
    den = add_(den, mul_((float)n_cos, cos_pdf(nh, d)));
    area = (ok && den > 0.f && den < INFINITY) ? div_((float)s.N, den) : 0.f;
    return d;
}

}  // namespace r3dg
