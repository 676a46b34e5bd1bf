/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * CPU restatement (plain C + OpenMP) of the reference rasterizer's algorithm, used only by
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs as the
 * checker.  Nothing under relightable3dgaussian_b200/ may call into this file.
 *
 * Parity status: PINNED — checked against outputs of the unmodified reference CUDA kernels
 * (oracle/_ref/libref_raster.so, built by oracle/build_ref.sh from /root/reference) on the GPU
 * box; the resulting golden vectors live in tests/golden/ (generator: tests/golden/make_golden.py).
 *
 * Every function cites the reference file:line it follows.  Floating point: the reference is
 * compiled with nvcc's default -fmad=true, which contracts a*b+c in NVVM *and* again in ptxas;
 * the association used below was read off the reference's sm_100 SASS with tools/sass_trace.py
 * (see DESIGN.md §"bit-exact binning") and is pinned with fmaf().  This file must be compiled
 * with -ffp-contract=off so that gcc adds no contraction of its own.  +,-,*,/,sqrt are IEEE in
 * both worlds, so depth keys, radii and tile rectangles are bit-identical to the GPU; expf() is
 * not (CUDA's expf is ~2 ulp, MUFU.EX2 based), so composited images agree to ~1e-6 and
 * n_contrib can differ at measure-zero threshold pixels.
 */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define BLOCK_X 16
#define BLOCK_Y 16

/* SH constants: cuda_rasterizer/auxiliary.h:21-39 (same values as utils/sh_utils.py:24-47) */
static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f,  -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};

/* a0*b0 + a1*b1 + a2*b2 as the reference binary evaluates every 3-term dot product:
 * the middle product is a plain multiply, then the first and third are fused onto it
 * (SASS: FMUL y; FFMA x; FFMA z). */
static inline float dot3(float a0, float b0, float a1, float b1, float a2, float b2) {
    return fmaf(a2, b2, fmaf(a0, b0, a1 * b1));
}

int oracle_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* transformPoint4x3 / 4x4 row: auxiliary.h:58-77.  m is the transposed (row-vector) matrix. */
static inline float xform_row(const float* m, int r, float x, float y, float z) {
    return dot3(x, m[r], y, m[4 + r], z, m[8 + r]) + m[12 + r];
}

/* float -> int as a CUDA (int) cast compiles (cvt.rzi.s32.f32): truncation, saturating at the int range, NaN -> 0.
 * A C cast is undefined there (x86 gives INT_MIN); the reference reaches NaN for the radius of a Gaussian whose 2D
 * covariance is negative definite (sqrt of a negative eigenvalue, forward.cu:231-233) and gets radius 0. */
static inline int f2i_rz(float v) {
    if (v != v) return 0;
    if (v >= 2147483648.0f) return INT_MAX;
    if (v <= -2147483648.0f) return INT_MIN;
    return (int)v;
}

/* getRect: auxiliary.h:46-56.  Division by BLOCK_X=16 is compiled to an exact *0.0625f. */
static inline void get_rect(float px, float py, int radius, int gx, int gy, int* x0, int* y0,
                            int* x1, int* y1) {
    float r = (float)radius;
    int a;
    a = f2i_rz((px - r) * 0.0625f);                    *x0 = a < 0 ? 0 : (a > gx ? gx : a);
    a = f2i_rz((py - r) * 0.0625f);                    *y0 = a < 0 ? 0 : (a > gy ? gy : a);
    a = f2i_rz((((px + r) + 16.0f) + -1.0f) * 0.0625f); *x1 = a < 0 ? 0 : (a > gx ? gx : a);
    a = f2i_rz((((py + r) + 16.0f) + -1.0f) * 0.0625f); *y1 = a < 0 ? 0 : (a > gy ? gy : a);
}

/* computeCov3D: forward.cu:119-153 (M = S*R in glm column-major, Sigma = M^T M; quaternion is
 * NOT normalised, forward.cu:128).  Includes the literal 0*x terms of the glm mat3 products —
 * they only matter for inf/NaN/-0 but keeping them keeps the restatement exact. */
static void cov3d_from_scale_rot(const float* s3, float mod, const float* q4, float* cov6) {
    const float r = q4[0], x = q4[1], y = q4[2], z = q4[3];
    const float sx = s3[0] * mod, sy = s3[1] * mod, sz = s3[2] * mod;
    const float yy = y * y, zz = z * z, xz = x * z, rx = r * x, rz = r * z;
    /* rotation entries (doubled sums) exactly as compiled */
    const float R00 = 1.0f - ((yy + zz) + (yy + zz));               /* 1-2(yy+zz) */
    const float t_xy_m = fmaf(x, y, -rz), R01 = t_xy_m + t_xy_m;     /* 2(xy-rz)   */
    const float t_xz_p = fmaf(r, y, xz), R02 = t_xz_p + t_xz_p;      /* 2(xz+ry)   */
    const float t_xy_p = fmaf(x, y, rz), R10 = t_xy_p + t_xy_p;      /* 2(xy+rz)   */
    const float t11 = fmaf(x, x, zz), R11 = 1.0f - (t11 + t11);      /* 1-2(xx+zz) */
    const float t_yz_m = fmaf(y, z, -rx), R12 = t_yz_m + t_yz_m;     /* 2(yz-rx)   */
    const float t_xz_m = fmaf(-r, y, xz), R20 = t_xz_m + t_xz_m;     /* 2(xz-ry)   */
    const float t_yz_p = fmaf(y, z, rx), R21 = t_yz_p + t_yz_p;      /* 2(yz+rx)   */
    const float t22 = fmaf(x, x, yy), R22 = 1.0f - (t22 + t22);      /* 1-2(xx+yy) */
    /* M = S * R (glm column-major product, zero terms kept).  Named by (glm column, row). */
    const float z00 = 0.0f * R00, z11 = 0.0f * R11, z21 = 0.0f * R21;
    /* The compiled form differs per column in which product is the plain multiply; restated 1:1. */
    const float m00 = fmaf(0.0f, R02, fmaf(0.0f, R01, sx * R00));   /* col0.x */
    const float m01 = fmaf(0.0f, R02, fmaf(sy, R01, z00));          /* col0.y */
    const float m02 = fmaf(sz, R02, fmaf(0.0f, R01, z00));          /* col0.z */
    const float m10 = fmaf(0.0f, R12, fmaf(sx, R10, z11));          /* col1.x */
    const float m11 = fmaf(0.0f, R12, fmaf(0.0f, R10, sy * R11));   /* col1.y */
    const float m12 = fmaf(sz, R12, fmaf(0.0f, R10, z11));          /* col1.z */
    const float m20 = fmaf(0.0f, R22, fmaf(sx, R20, z21));          /* col2.x */
    const float m21 = fmaf(0.0f, R22, fmaf(0.0f, R20, sy * R21));   /* col2.y */
    const float m22 = fmaf(sz, R22, fmaf(0.0f, R20, z21));          /* col2.z */
    /* Sigma = M^T M : dot of columns, y-first association */
    cov6[0] = dot3(m00, m00, m01, m01, m02, m02);
    cov6[1] = dot3(m00, m10, m01, m11, m02, m12);
    cov6[2] = dot3(m00, m20, m01, m21, m02, m22);
    cov6[3] = dot3(m10, m10, m11, m11, m12, m12);
    cov6[4] = dot3(m10, m20, m11, m21, m12, m22);
    cov6[5] = dot3(m20, m20, m21, m21, m22, m22);
}

/* computeColorFromSH: forward.cu:20-71.  Not on the bit-exact path (tolerance 1e-4), association
 * follows the compiled kernel anyway (one running fma chain per channel). */
static void sh_to_rgb(int deg, const float* pos, const float* campos, const float* sh /*[M][3]*/,
                      float* rgb, uint8_t* clamped) {
    float dx = pos[0] - campos[0], dy = pos[1] - campos[1], dz = pos[2] - campos[2];
    float len = sqrtf(dot3(dx, dx, dy, dy, dz, dz));
    float x = dx / len, y = dy / len, z = dz / len;
    float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    for (int c = 0; c < 3; ++c) {
        float res = SH_C0 * sh[0 * 3 + c];
        if (deg > 0) {
            res = fmaf(-(SH_C1 * y), sh[1 * 3 + c], res);
            res = fmaf(SH_C1 * z, sh[2 * 3 + c], res);
            res = fmaf(-(SH_C1 * x), sh[3 * 3 + c], res);
            if (deg > 1) {
                res = fmaf(SH_C2[0] * xy, sh[4 * 3 + c], res);
                res = fmaf(SH_C2[1] * yz, sh[5 * 3 + c], res);
                res = fmaf(SH_C2[2] * ((zz + zz) - xx - yy), sh[6 * 3 + c], res);
                res = fmaf(SH_C2[3] * xz, sh[7 * 3 + c], res);
                res = fmaf(SH_C2[4] * (xx - yy), sh[8 * 3 + c], res);
                if (deg > 2) {
                    res = fmaf(SH_C3[0] * y * fmaf(xx, 3.0f, -yy), sh[9 * 3 + c], res);
                    res = fmaf(SH_C3[1] * xy * z, sh[10 * 3 + c], res);
                    res = fmaf(SH_C3[2] * y * (fmaf(zz, 4.0f, -xx) - yy), sh[11 * 3 + c], res);
                    res = fmaf(SH_C3[3] * z * fmaf(yy, -3.0f, fmaf(xx, -3.0f, zz + zz)),
                               sh[12 * 3 + c], res);
                    res = fmaf(SH_C3[4] * x * (fmaf(zz, 4.0f, -xx) - yy), sh[13 * 3 + c], res);
                    res = fmaf(SH_C3[5] * z * (xx - yy), sh[14 * 3 + c], res);
                    res = fmaf(SH_C3[6] * x * fmaf(yy, -3.0f, xx), sh[15 * 3 + c], res);
                }
            }
        }
        res += 0.5f;
        clamped[c] = res < 0.0f;
        rgb[c] = res < 0.0f ? 0.0f : res;
    }
}

/* preprocessCUDA (forward): forward.cu:156-258, in_frustum auxiliary.h:139-164,
 * computeCov2D forward.cu:74-113, ndc2Pix auxiliary.h:41-44.
 * Outputs (all sized P): radii, means2D[2P], depths, cov3D[6P], conic_opacity[4P], rgb[3P],
 * clamped[3P], tiles_touched.  Untouched entries keep the caller's initial values, like the
 * reference (which only zero-inits radii and tiles_touched). */
void oracle_preprocess(int P, int D, int M, const float* means3D, const float* scales,
                       float scale_modifier, const float* rotations, const float* opacities,
                       const float* shs, const float* cov3D_precomp, const float* colors_precomp,
                       const float* viewmatrix, const float* projmatrix, const float* campos, int W,
                       int H, float tan_fovx, float tan_fovy, int* radii, float* means2D,
                       float* depths, float* cov3Ds, float* conic_opacity, float* rgb,
                       uint8_t* clamped, uint32_t* tiles_touched) {
    const float focal_y = H / (2.0f * tan_fovy);   /* rasterizer_impl.cu:232-233 */
    const float focal_x = W / (2.0f * tan_fovx);
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    const float* V = viewmatrix;
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; ++idx) {
        radii[idx] = 0;
        tiles_touched[idx] = 0;
        const float px = means3D[3 * idx], py = means3D[3 * idx + 1], pz = means3D[3 * idx + 2];
        const float tz = xform_row(V, 2, px, py, pz);         /* p_view.z */
        if (tz <= 0.2f) continue;                             /* auxiliary.h:154 */
        const float hx = xform_row(projmatrix, 0, px, py, pz);
        const float hy = xform_row(projmatrix, 1, px, py, pz);
        const float hw = xform_row(projmatrix, 3, px, py, pz);
        const float p_w = 1.0f / (hw + 0.0000001f);
        const float projx = hx * p_w, projy = hy * p_w;

        float c6[6];
        if (cov3D_precomp) {
            memcpy(c6, cov3D_precomp + 6 * idx, sizeof c6);
        } else {
            cov3d_from_scale_rot(scales + 3 * idx, scale_modifier, rotations + 4 * idx, c6);
            memcpy(cov3Ds + 6 * idx, c6, sizeof c6);
        }
        /* computeCov2D */
        const float tx = xform_row(V, 0, px, py, pz), ty = xform_row(V, 1, px, py, pz);
        const float limx = tan_fovx * 1.3f, limy = tan_fovy * 1.3f;
        const float cxz = fminf(fmaxf(tx / tz, -limx), limx);
        const float cyz = fminf(fmaxf(ty / tz, -limy), limy);
        const float tz2 = tz * tz;
        /* J entries: focal/tz and -(focal * (clamp*tz)) / tz^2; the sign is folded into the
         * clamp product by the compiler (exact). */
        const float j00 = focal_x / tz, j11 = focal_y / tz;
        const float j02 = ((tz * -cxz) * focal_x) / tz2;
        const float j12 = ((tz * -cyz) * focal_y) / tz2;
        /* T = W * J (glm), rows 0/1 of T^T:  T0[k] = W[k][0]*j00 + 0*W[k][1] + W[k][2]*j02 */
        float T0[3], T1[3];
        for (int k = 0; k < 3; ++k) {
            const float w0 = V[4 * k + 0], w1 = V[4 * k + 1], w2 = V[4 * k + 2];
            T0[k] = fmaf(w2, j02, fmaf(w0, j00, 0.0f * w1));
            T1[k] = fmaf(w2, j12, fmaf(0.0f, w0, w1 * j11));
        }
        /* Vrk * T columns, then T^T * (.) ; all y-first dot3 */
        const float a0 = dot3(T0[0], c6[0], T0[1], c6[1], T0[2], c6[2]);
        const float a1 = dot3(T0[0], c6[1], T0[1], c6[3], T0[2], c6[4]);
        const float a2 = dot3(T0[0], c6[2], T0[1], c6[4], T0[2], c6[5]);
        const float b0 = dot3(T1[0], c6[0], T1[1], c6[1], T1[2], c6[2]);
        const float b1 = dot3(T1[0], c6[1], T1[1], c6[3], T1[2], c6[4]);
        const float b2 = dot3(T1[0], c6[2], T1[1], c6[4], T1[2], c6[5]);
        const float cov_a = dot3(T0[0], a0, T0[1], a1, T0[2], a2) + 0.3f;
        const float cov_c = dot3(T1[0], b0, T1[1], b1, T1[2], b2) + 0.3f;
        const float cov_b = dot3(T0[0], b0, T0[1], b1, T0[2], b2);

        const float det = fmaf(cov_a, cov_c, -(cov_b * cov_b));
        if (det == 0.0f) continue;
        const float det_inv = 1.0f / det;
        const float con_a = cov_c * det_inv, con_b = cov_b * -det_inv, con_c = cov_a * det_inv;
        const float mid = (cov_a + cov_c) * 0.5f;
        const float disc = sqrtf(fmaxf(fmaf(mid, mid, -det), 0.1f));
        const float lam = fmaxf(mid + disc, mid - disc);
        const int my_radius = f2i_rz(ceilf(sqrtf(lam) * 3.0f));
        const float pix_x = (float)(fma((double)projx + 1.0, (double)W, -1.0) * 0.5);
        const float pix_y = (float)(fma((double)projy + 1.0, (double)H, -1.0) * 0.5);
        int x0, y0, x1, y1;
        get_rect(pix_x, pix_y, my_radius, gx, gy, &x0, &y0, &x1, &y1);
        if ((x1 - x0) * (y1 - y0) == 0) continue;

        if (!colors_precomp)
            sh_to_rgb(D, means3D + 3 * idx, campos, shs + (size_t)idx * M * 3, rgb + 3 * idx,
                      clamped + 3 * idx);
        depths[idx] = tz;
        radii[idx] = my_radius;
        means2D[2 * idx] = pix_x;
        means2D[2 * idx + 1] = pix_y;
        conic_opacity[4 * idx + 0] = con_a;
        conic_opacity[4 * idx + 1] = con_b;
        conic_opacity[4 * idx + 2] = con_c;
        conic_opacity[4 * idx + 3] = opacities[idx];
        tiles_touched[idx] = (uint32_t)((y1 - y0) * (x1 - x0));
    }
}

/* checkFrustum / markVisible: rasterizer_impl.cu:54-66,141-153 */
void oracle_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present) {
    for (int i = 0; i < P; ++i)
        present[i] = xform_row(viewmatrix, 2, means3D[3 * i], means3D[3 * i + 1],
                               means3D[3 * i + 2]) > 0.2f;
}

/* Stable LSD radix sort of (u64 key, u32 value) on bits [0, end_bit): the semantics of
 * cub::DeviceRadixSort::SortPairs at rasterizer_impl.cu:313-318. */
static void radix_sort_pairs(uint64_t* keys, uint32_t* vals, uint64_t* ktmp, uint32_t* vtmp,
                             size_t n, int end_bit) {
    for (int shift = 0; shift < end_bit; shift += 8) {
        size_t hist[257] = {0};
        int bits = end_bit - shift < 8 ? end_bit - shift : 8;
        uint64_t mask = (1u << bits) - 1;
        for (size_t i = 0; i < n; ++i) hist[((keys[i] >> shift) & mask) + 1]++;
        for (int d = 0; d < 256; ++d) hist[d + 1] += hist[d];
        for (size_t i = 0; i < n; ++i) {
            size_t p = hist[(keys[i] >> shift) & mask]++;
            ktmp[p] = keys[i];
            vtmp[p] = vals[i];
        }
        uint64_t* kt = keys; keys = ktmp; ktmp = kt;
        uint32_t* vt = vals; vals = vtmp; vtmp = vt;
    }
    int passes = (end_bit + 7) / 8;
    if (passes & 1) {  /* result currently lives in the scratch pair */
        memcpy(ktmp, keys, n * sizeof(uint64_t));
        memcpy(vtmp, vals, n * sizeof(uint32_t));
    }
}

/* getHigherMsb: rasterizer_impl.cu:35-50 */
static uint32_t higher_msb(uint32_t n) {
    uint32_t msb = sizeof(n) * 4, step = msb;
    while (step > 1) {
        step /= 2;
        if (n >> msb) msb += step; else msb -= step;
    }
    if (n >> msb) msb++;
    return msb;
}

/* InclusiveSum + duplicateWithKeys + SortPairs + identifyTileRanges:
 * rasterizer_impl.cu:287,70-111,310-318,116-138,320-327.
 * point_offsets[P] out; returns R.  keys/point_list must hold R entries: call once with
 * keys==NULL to get R. ranges is uint2[T] (zero-filled here). */
int64_t oracle_bin(int P, int W, int H, const int* radii, const float* means2D,
                   const float* depths, const uint32_t* tiles_touched, uint32_t* point_offsets,
                   uint64_t* keys_sorted, uint32_t* point_list, uint32_t* ranges) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    uint32_t acc = 0;
    for (int i = 0; i < P; ++i) { acc += tiles_touched[i]; point_offsets[i] = acc; }
    const size_t R = acc;
    if (!keys_sorted) return (int64_t)R;
    uint64_t* ktmp = (uint64_t*)malloc((R + 1) * sizeof(uint64_t));
    uint32_t* vtmp = (uint32_t*)malloc((R + 1) * sizeof(uint32_t));
    for (int idx = 0; idx < P; ++idx) {
        if (radii[idx] <= 0) continue;
        uint32_t off = idx == 0 ? 0 : point_offsets[idx - 1];
        int x0, y0, x1, y1;
        get_rect(means2D[2 * idx], means2D[2 * idx + 1], radii[idx], gx, gy, &x0, &y0, &x1, &y1);
        uint32_t dbits;
        memcpy(&dbits, depths + idx, 4);
        for (int y = y0; y < y1; ++y)
            for (int x = x0; x < x1; ++x) {
                uint64_t key = (uint64_t)(y * gx + x);
                key <<= 32;
                key |= dbits;
                keys_sorted[off] = key;
                point_list[off] = (uint32_t)idx;
                off++;
            }
    }
    radix_sort_pairs(keys_sorted, point_list, ktmp, vtmp, R, 32 + (int)higher_msb(gx * gy));
    free(ktmp); free(vtmp);
    memset(ranges, 0, (size_t)gx * gy * 2 * sizeof(uint32_t));
    for (size_t i = 0; i < R; ++i) {
        uint32_t cur = (uint32_t)(keys_sorted[i] >> 32);
        if (i == 0) ranges[2 * cur] = 0;
        else {
            uint32_t prev = (uint32_t)(keys_sorted[i - 1] >> 32);
            if (cur != prev) { ranges[2 * prev + 1] = (uint32_t)i; ranges[2 * cur] = (uint32_t)i; }
        }
        if (i == R - 1) ranges[2 * cur + 1] = (uint32_t)R;
    }
    return (int64_t)R;
}

/* renderCUDA forward: forward.cu:263-395.  One task per tile, pixels sequential.
 * colors: [P,3]; features: [P,S]; outputs planar CHW.  out_weights must be zero-initialised. */
void oracle_render_forward(int W, int H, int S, const uint32_t* ranges, const uint32_t* point_list,
                           const float* means2D, const float* depths, const float* features,
                           const float* colors, const float* conic_opacity, const float* bg,
                           float* final_T, uint32_t* n_contrib, float* out_color,
                           float* out_opacity, float* out_depth, float* out_feature,
                           float* out_weights) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    const size_t HW = (size_t)H * W;
#pragma omp parallel for schedule(dynamic, 1)
    for (int tile = 0; tile < gx * gy; ++tile) {
        const int tx = tile % gx, ty = tile / gx;
        const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int ly = 0; ly < BLOCK_Y; ++ly)
            for (int lx = 0; lx < BLOCK_X; ++lx) {
                const int pxi = tx * BLOCK_X + lx, pyi = ty * BLOCK_Y + ly;
                if (pxi >= W || pyi >= H) continue;
                const size_t pix = (size_t)W * pyi + pxi;
                const float pxf = (float)pxi, pyf = (float)pyi;
                float T = 1.0f, C[3] = {0, 0, 0}, F[64] = {0}, Dp = 0.0f, Op = 0.0f;
                uint32_t contributor = 0, last = 0;
                for (uint32_t k = r0; k < r1; ++k) {
                    contributor++;
                    const uint32_t id = point_list[k];
                    const float dx = means2D[2 * id] - pxf, dy = means2D[2 * id + 1] - pyf;
                    const float ca = conic_opacity[4 * id], cb = conic_opacity[4 * id + 1],
                                cc = conic_opacity[4 * id + 2], op = conic_opacity[4 * id + 3];
                    /* power = -0.5f*(ca*dx*dx + cc*dy*dy) - cb*dx*dy, forward.cu:344, as compiled */
                    const float q = fmaf(dx, dx * ca, dy * (dy * cc));
                    const float power = fmaf(q, -0.5f, -(dy * (dx * cb)));
                    if (power > 0.0f) continue;
                    const float alpha = fminf(0.99f, op * expf(power));
                    if (alpha < 1.0f / 255.0f) continue;
                    const float test_T = T * (1.0f - alpha);
                    if (test_T < 0.0001f) break;   /* done = true; nothing after it counts */
                    const float w = T * alpha;
                    for (int ch = 0; ch < 3; ++ch) C[ch] = fmaf(w, colors[3 * id + ch], C[ch]);
                    for (int ch = 0; ch < S; ++ch) F[ch] = fmaf(w, features[(size_t)id * S + ch], F[ch]);
                    Dp = fmaf(w, depths[id], Dp);
                    Op = Op + w;
                    T = test_T;
#pragma omp atomic
                    out_weights[id] += w;
                    last = contributor;
                }
                final_T[pix] = T;
                n_contrib[pix] = last;
                for (int ch = 0; ch < 3; ++ch) out_color[ch * HW + pix] = fmaf(bg[ch], T, C[ch]);
                for (int ch = 0; ch < S; ++ch) out_feature[ch * HW + pix] = F[ch];
                out_depth[pix] = Dp;
                out_opacity[pix] = Op;
            }
    }
}

/* renderSurfaceXYZCUDA + renderPseudoNormalCUDA: forward.cu:398-491.  out_normal must be
 * zero-initialised (pixels with zero-length normals are left untouched, forward.cu:480-482). */
void oracle_surface_normal(int W, int H, const float* viewmatrix, float tan_fovx, float tan_fovy,
                           float cx, float cy, const float* opacity, const float* depth,
                           float* out_normal, float* out_xyz) {
    const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
    const size_t HW = (size_t)H * W;
    const float* V = viewmatrix;
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            const size_t p = (size_t)W * y + x;
            const float d = depth[p] / fmaxf(opacity[p], 0.0000001f);
            out_xyz[p] = (((float)x - cx) / focal_x) * d;
            out_xyz[HW + p] = (((float)y - cy) / focal_y) * d;
            out_xyz[2 * HW + p] = d;
        }
#pragma omp parallel for schedule(static)
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            const int xm = x == 0 ? 0 : x - 1, xp = x == W - 1 ? W - 1 : x + 1;
            const int ym = y == 0 ? 0 : y - 1, yp = y == H - 1 ? H - 1 : y + 1;
            float ga[3], gb[3];
            for (int i = 0; i < 3; ++i) {
                const float* s = out_xyz + i * HW;
                const float x00 = s[(size_t)W * ym + xm], x01 = s[(size_t)W * ym + x],
                            x02 = s[(size_t)W * ym + xp], x10 = s[(size_t)W * y + xm],
                            x12 = s[(size_t)W * y + xp], x20 = s[(size_t)W * yp + xm],
                            x21 = s[(size_t)W * yp + x], x22 = s[(size_t)W * yp + xp];
                const float h = x00 * -0.125f;
                ga[i] = fmaf(x22, 0.125f, fmaf(x20, -0.125f, fmaf(x12, 0.25f,
                        fmaf(x10, -0.25f, fmaf(x02, 0.125f, h)))));
                gb[i] = fmaf(x22, 0.125f, fmaf(x21, 0.25f, fmaf(x20, 0.125f,
                        fmaf(x02, -0.125f, fmaf(x01, -0.25f, h)))));
            }
            const float n0 = fmaf(ga[1], gb[2], -(ga[2] * gb[1]));
            const float n1 = fmaf(ga[2], gb[0], -(ga[0] * gb[2]));
            const float n2 = fmaf(ga[0], gb[1], -(ga[1] * gb[0]));
            const float norm = sqrtf(fmaf(n2, n2, fmaf(n0, n0, n1 * n1)));
            if (norm <= 0.0f) continue;
            const float N0 = -n0 / norm, N1 = -n1 / norm, N2 = -n2 / norm;
            const size_t p = (size_t)W * y + x;
            out_normal[p] = dot3(V[0], N0, V[1], N1, V[2], N2);
            out_normal[HW + p] = dot3(V[4], N0, V[5], N1, V[6], N2);
            out_normal[2 * HW + p] = dot3(V[8], N0, V[9], N1, V[10], N2);
        }
}

static inline void atomic_addf(float* p, float v) {
#pragma omp atomic
    *p += v;
}

/* renderCUDA backward: backward.cu:401-614.  All dL_* outputs must be zero-initialised.
 * dL_dmean2D is [P,3] (depth gradient in .z), dL_dconic is [P,4] (x,y,_,w used). */
void oracle_render_backward(int W, int H, int S, const uint32_t* ranges,
                            const uint32_t* point_list, const float* bg, const float* means2D,
                            const float* depths, const float* conic_opacity, const float* colors,
                            const float* features, const float* final_T, const uint32_t* n_contrib,
                            const float* dL_dpix, const float* dL_dpix_o, const float* dL_dpix_d,
                            const float* dL_dpix_f, int backward_geometry, float* dL_dmean2D,
                            float* dL_dconic, float* dL_dopacity, float* dL_dcolors,
                            float* dL_dfeature) {
    const int gx = (W + BLOCK_X - 1) / BLOCK_X, gy = (H + BLOCK_Y - 1) / BLOCK_Y;
    const size_t HW = (size_t)H * W;
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;
#pragma omp parallel for schedule(dynamic, 1)
    for (int tile = 0; tile < gx * gy; ++tile) {
        const int tx = tile % gx, ty = tile / gx;
        const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int ly = 0; ly < BLOCK_Y; ++ly)
            for (int lx = 0; lx < BLOCK_X; ++lx) {
                const int pxi = tx * BLOCK_X + lx, pyi = ty * BLOCK_Y + ly;
                if (pxi >= W || pyi >= H) continue;
                const size_t pix = (size_t)W * pyi + pxi;
                const float pxf = (float)pxi, pyf = (float)pyi;
                const float T_final = final_T[pix];
                float T = T_final;
                const uint32_t last_contributor = n_contrib[pix];
                float accum_rec[3] = {0}, accum_rec_d = 0, accum_rec_o = 0, accum_rec_f[64] = {0};
                float dpix[3], dpix_f[64];
                for (int c = 0; c < 3; ++c) dpix[c] = dL_dpix[c * HW + pix];
                const float dpix_d = dL_dpix_d[pix], dpix_o = dL_dpix_o[pix];
                for (int c = 0; c < S; ++c) dpix_f[c] = dL_dpix_f[c * HW + pix];
                float last_alpha = 0, last_depth = 0, last_color[3] = {0}, last_feature[64] = {0};
                float bg_dot = 0;
                for (int c = 0; c < 3; ++c) bg_dot += bg[c] * dpix[c];
                /* back to front; entry k (0-based from r0) has contributor index k+1 */
                for (uint32_t k = r1; k-- > r0;) {
                    const uint32_t contributor = k - r0;       /* after the reference's -- */
                    if (contributor >= last_contributor) continue;
                    const uint32_t id = point_list[k];
                    const float dx = means2D[2 * id] - pxf, dy = means2D[2 * id + 1] - pyf;
                    const float ca = conic_opacity[4 * id], cb = conic_opacity[4 * id + 1],
                                cc = conic_opacity[4 * id + 2], op = conic_opacity[4 * id + 3];
                    const float q = fmaf(dx, dx * ca, dy * (dy * cc));
                    const float power = fmaf(q, -0.5f, -(dy * (dx * cb)));
                    if (power > 0.0f) continue;
                    const float G = expf(power);
                    const float alpha = fminf(0.99f, op * G);
                    if (alpha < 1.0f / 255.0f) continue;
                    T = T / (1.0f - alpha);
                    const float dchannel_dcolor = alpha * T;
                    float dL_dalpha = 0.0f;
                    for (int ch = 0; ch < 3; ++ch) {
                        const float c = colors[3 * id + ch];
                        accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
                        last_color[ch] = c;
                        dL_dalpha += (c - accum_rec[ch]) * dpix[ch];
                        atomic_addf(&dL_dcolors[3 * id + ch], dchannel_dcolor * dpix[ch]);
                    }
                    for (int ch = 0; ch < S; ++ch) {
                        const float f = features[(size_t)id * S + ch];
                        accum_rec_f[ch] = last_alpha * last_feature[ch] + (1.f - last_alpha) * accum_rec_f[ch];
                        last_feature[ch] = f;
                        if (backward_geometry) dL_dalpha += (f - accum_rec_f[ch]) * dpix_f[ch];
                        atomic_addf(&dL_dfeature[(size_t)id * S + ch], dchannel_dcolor * dpix_f[ch]);
                    }
                    const float depth = depths[id];
                    accum_rec_d = last_alpha * last_depth + (1.f - last_alpha) * accum_rec_d;
                    last_depth = depth;
                    dL_dalpha += (depth - accum_rec_d) * dpix_d;
                    accum_rec_o = last_alpha + (1.f - last_alpha) * accum_rec_o;
                    dL_dalpha += (1.0f - accum_rec_o) * dpix_o;
                    dL_dalpha *= T;
                    last_alpha = alpha;
                    dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
                    const float dL_dG = op * dL_dalpha;
                    const float gdx = G * dx, gdy = G * dy;
                    const float dG_ddelx = -gdx * ca - gdy * cb;
                    const float dG_ddely = -gdy * cc - gdx * cb;
                    atomic_addf(&dL_dmean2D[3 * id + 0], dL_dG * dG_ddelx * ddelx_dx);
                    atomic_addf(&dL_dmean2D[3 * id + 1], dL_dG * dG_ddely * ddely_dy);
                    atomic_addf(&dL_dmean2D[3 * id + 2], dpix_d * dchannel_dcolor);
                    atomic_addf(&dL_dconic[4 * id + 0], -0.5f * gdx * dx * dL_dG);
                    atomic_addf(&dL_dconic[4 * id + 1], -0.5f * gdx * dy * dL_dG);
                    atomic_addf(&dL_dconic[4 * id + 3], -0.5f * gdy * dy * dL_dG);
                    atomic_addf(&dL_dopacity[id], G * dL_dalpha);
                }
            }
    }
}

/* computeCov2DCUDA (backward.cu:144-276) + preprocessCUDA backward (backward.cu:348-398)
 * + computeColorFromSH backward (backward.cu:20-139) + computeCov3D backward
 * (backward.cu:280-343).  Gradient path: tolerance 1e-3 rel, natural association.
 * dL_dcolor [P,3] in; dL_dmeans [P,3], dL_dcov [P,6], dL_dsh [P,M,3], dL_dscale [P,3],
 * dL_drot [P,4] out (zero-initialised by caller). */
void oracle_preprocess_backward(int P, int D, int M, const float* means3D, const int* radii,
                                const float* shs, const uint8_t* clamped, const float* scales,
                                const float* rotations, float scale_modifier, const float* cov3Ds,
                                const float* viewmatrix, const float* projmatrix, int W, int H,
                                float tan_fovx, float tan_fovy, const float* campos,
                                const float* dL_dmean2D, const float* dL_dconic,
                                const float* dL_dcolor, float* dL_dmeans, float* dL_dcov,
                                float* dL_dsh, float* dL_dscale, float* dL_drot) {
    const float h_y = H / (2.0f * tan_fovy), h_x = W / (2.0f * tan_fovx);
    const float* V = viewmatrix;
    const float* proj = projmatrix;
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; ++idx) {
        if (!(radii[idx] > 0)) continue;
        const float* cov3D = cov3Ds + 6 * idx;
        const float mx = means3D[3 * idx], my = means3D[3 * idx + 1], mz = means3D[3 * idx + 2];
        const float dcx = dL_dconic[4 * idx], dcy = dL_dconic[4 * idx + 1], dcz = dL_dconic[4 * idx + 3];
        float t[3] = {V[0] * mx + V[4] * my + V[8] * mz + V[12], V[1] * mx + V[5] * my + V[9] * mz + V[13],
                      V[2] * mx + V[6] * my + V[10] * mz + V[14]};
        const float limx = 1.3f * tan_fovx, limy = 1.3f * tan_fovy;
        const float txtz = t[0] / t[2], tytz = t[1] / t[2];
        t[0] = fminf(limx, fmaxf(-limx, txtz)) * t[2];
        t[1] = fminf(limy, fmaxf(-limy, tytz)) * t[2];
        const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        /* glm column-major: J[col][row]; J = mat3(h_x/tz,0,-(h_x tx)/tz², 0,h_y/tz,-(h_y ty)/tz², 0,0,0) */
        const float J[3][3] = {{h_x / t[2], 0.f, -(h_x * t[0]) / (t[2] * t[2])},
                               {0.f, h_y / t[2], -(h_y * t[1]) / (t[2] * t[2])},
                               {0.f, 0.f, 0.f}};
        const float Wm[3][3] = {{V[0], V[4], V[8]}, {V[1], V[5], V[9]}, {V[2], V[6], V[10]}};
        const float Vrk[3][3] = {{cov3D[0], cov3D[1], cov3D[2]}, {cov3D[1], cov3D[3], cov3D[4]},
                                 {cov3D[2], cov3D[4], cov3D[5]}};
        float T[3][3]; /* T = W * J, glm: T[c][r] = sum_k W[k][r] * J[c][k] */
        for (int c = 0; c < 3; ++c)
            for (int r = 0; r < 3; ++r)
                T[c][r] = Wm[0][r] * J[c][0] + Wm[1][r] * J[c][1] + Wm[2][r] * J[c][2];
        /* cov2D = T^T * Vrk^T * T ; cov2D[c][r] = sum_ij T[r][i]... computed via helper */
        float VT[3][3]; /* (Vrk^T * T)[c][r] = sum_k Vrk^T[k][r] * T[c][k] = sum_k Vrk[r][k]*T[c][k] */
        for (int c = 0; c < 3; ++c)
            for (int r = 0; r < 3; ++r)
                VT[c][r] = Vrk[r][0] * T[c][0] + Vrk[r][1] * T[c][1] + Vrk[r][2] * T[c][2];
        /* (T^T * X)[c][r] = sum_k T^T[k][r] * X[c][k] = sum_k T[r][k] * X[c][k] */
        const float a = (T[0][0] * VT[0][0] + T[0][1] * VT[0][1] + T[0][2] * VT[0][2]) + 0.3f;
        const float b = T[1][0] * VT[0][0] + T[1][1] * VT[0][1] + T[1][2] * VT[0][2];
        const float c_ = (T[1][0] * VT[1][0] + T[1][1] * VT[1][1] + T[1][2] * VT[1][2]) + 0.3f;
        const float denom = a * c_ - b * b;
        float dL_da = 0, dL_db = 0, dL_dc = 0;
        const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
        float* dcov = dL_dcov + 6 * idx;
        if (denom2inv != 0) {
            dL_da = denom2inv * (-c_ * c_ * dcx + 2 * b * c_ * dcy + (denom - a * c_) * dcz);
            dL_dc = denom2inv * (-a * a * dcz + 2 * a * b * dcy + (denom - a * c_) * dcx);
            dL_db = denom2inv * 2 * (b * c_ * dcx - (denom + 2 * b * b) * dcy + a * b * dcz);
            dcov[0] = (T[0][0] * T[0][0] * dL_da + T[0][0] * T[1][0] * dL_db + T[1][0] * T[1][0] * dL_dc);
            dcov[3] = (T[0][1] * T[0][1] * dL_da + T[0][1] * T[1][1] * dL_db + T[1][1] * T[1][1] * dL_dc);
            dcov[5] = (T[0][2] * T[0][2] * dL_da + T[0][2] * T[1][2] * dL_db + T[1][2] * T[1][2] * dL_dc);
            dcov[1] = 2 * T[0][0] * T[0][1] * dL_da + (T[0][0] * T[1][1] + T[0][1] * T[1][0]) * dL_db + 2 * T[1][0] * T[1][1] * dL_dc;
            dcov[2] = 2 * T[0][0] * T[0][2] * dL_da + (T[0][0] * T[1][2] + T[0][2] * T[1][0]) * dL_db + 2 * T[1][0] * T[1][2] * dL_dc;
            dcov[4] = 2 * T[0][2] * T[0][1] * dL_da + (T[0][1] * T[1][2] + T[0][2] * T[1][1]) * dL_db + 2 * T[1][1] * T[1][2] * dL_dc;
        } else {
            for (int i = 0; i < 6; ++i) dcov[i] = 0;
        }
        const float dL_dT00 = 2 * (T[0][0] * Vrk[0][0] + T[0][1] * Vrk[0][1] + T[0][2] * Vrk[0][2]) * dL_da +
                              (T[1][0] * Vrk[0][0] + T[1][1] * Vrk[0][1] + T[1][2] * Vrk[0][2]) * dL_db;
        const float dL_dT01 = 2 * (T[0][0] * Vrk[1][0] + T[0][1] * Vrk[1][1] + T[0][2] * Vrk[1][2]) * dL_da +
                              (T[1][0] * Vrk[1][0] + T[1][1] * Vrk[1][1] + T[1][2] * Vrk[1][2]) * dL_db;
        const float dL_dT02 = 2 * (T[0][0] * Vrk[2][0] + T[0][1] * Vrk[2][1] + T[0][2] * Vrk[2][2]) * dL_da +
                              (T[1][0] * Vrk[2][0] + T[1][1] * Vrk[2][1] + T[1][2] * Vrk[2][2]) * dL_db;
        const float dL_dT10 = 2 * (T[1][0] * Vrk[0][0] + T[1][1] * Vrk[0][1] + T[1][2] * Vrk[0][2]) * dL_dc +
                              (T[0][0] * Vrk[0][0] + T[0][1] * Vrk[0][1] + T[0][2] * Vrk[0][2]) * dL_db;
        const float dL_dT11 = 2 * (T[1][0] * Vrk[1][0] + T[1][1] * Vrk[1][1] + T[1][2] * Vrk[1][2]) * dL_dc +
                              (T[0][0] * Vrk[1][0] + T[0][1] * Vrk[1][1] + T[0][2] * Vrk[1][2]) * dL_db;
        const float dL_dT12 = 2 * (T[1][0] * Vrk[2][0] + T[1][1] * Vrk[2][1] + T[1][2] * Vrk[2][2]) * dL_dc +
                              (T[0][0] * Vrk[2][0] + T[0][1] * Vrk[2][1] + T[0][2] * Vrk[2][2]) * dL_db;
        const float dL_dJ00 = Wm[0][0] * dL_dT00 + Wm[0][1] * dL_dT01 + Wm[0][2] * dL_dT02;
        const float dL_dJ02 = Wm[2][0] * dL_dT00 + Wm[2][1] * dL_dT01 + Wm[2][2] * dL_dT02;
        const float dL_dJ11 = Wm[1][0] * dL_dT10 + Wm[1][1] * dL_dT11 + Wm[1][2] * dL_dT12;
        const float dL_dJ12 = Wm[2][0] * dL_dT10 + Wm[2][1] * dL_dT11 + Wm[2][2] * dL_dT12;
        const float tz = 1.f / t[2], tz2 = tz * tz, tz3 = tz2 * tz;
        const float dL_dtx = x_grad_mul * -h_x * tz2 * dL_dJ02;
        const float dL_dty = y_grad_mul * -h_y * tz2 * dL_dJ12;
        const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * t[0]) * tz3 * dL_dJ02 +
                             (2 * h_y * t[1]) * tz3 * dL_dJ12;
        const float gz = dL_dtz + dL_dmean2D[3 * idx + 2];
        float dmean[3] = {V[0] * dL_dtx + V[1] * dL_dty + V[2] * gz, V[4] * dL_dtx + V[5] * dL_dty + V[6] * gz,
                          V[8] * dL_dtx + V[9] * dL_dty + V[10] * gz};   /* assigned, backward.cu:275 */

        /* preprocessCUDA backward: backward.cu:372-389 */
        const float m_hom_w = proj[3] * mx + proj[7] * my + proj[11] * mz + proj[15];
        const float m_w = 1.0f / (m_hom_w + 0.0000001f);
        const float mul1 = (proj[0] * mx + proj[4] * my + proj[8] * mz + proj[12]) * m_w * m_w;
        const float mul2 = (proj[1] * mx + proj[5] * my + proj[9] * mz + proj[13]) * m_w * m_w;
        const float g2x = dL_dmean2D[3 * idx], g2y = dL_dmean2D[3 * idx + 1];
        dmean[0] += (proj[0] * m_w - proj[3] * mul1) * g2x + (proj[1] * m_w - proj[3] * mul2) * g2y;
        dmean[1] += (proj[4] * m_w - proj[7] * mul1) * g2x + (proj[5] * m_w - proj[7] * mul2) * g2y;
        dmean[2] += (proj[8] * m_w - proj[11] * mul1) * g2x + (proj[9] * m_w - proj[11] * mul2) * g2y;

        if (shs) { /* backward.cu:20-139 */
            const float dox = mx - campos[0], doy = my - campos[1], doz = mz - campos[2];
            const float len = sqrtf(dox * dox + doy * doy + doz * doz);
            const float x = dox / len, y = doy / len, z = doz / len;
            const float* sh = shs + (size_t)idx * M * 3;
            float* dsh = dL_dsh + (size_t)idx * M * 3;
            float dRGB[3], dRGBdx[3] = {0}, dRGBdy[3] = {0}, dRGBdz[3] = {0};
            for (int c = 0; c < 3; ++c) dRGB[c] = dL_dcolor[3 * idx + c] * (clamped[3 * idx + c] ? 0.f : 1.f);
#define SHC(k, c) sh[(k) * 3 + (c)]
#define DSH(k, w) for (int c = 0; c < 3; ++c) dsh[(k) * 3 + c] = (w) * dRGB[c]
            DSH(0, SH_C0);
            if (D > 0) {
                DSH(1, -SH_C1 * y); DSH(2, SH_C1 * z); DSH(3, -SH_C1 * x);
                for (int c = 0; c < 3; ++c) {
                    dRGBdx[c] = -SH_C1 * SHC(3, c); dRGBdy[c] = -SH_C1 * SHC(1, c); dRGBdz[c] = SH_C1 * SHC(2, c);
                }
                if (D > 1) {
                    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    DSH(4, SH_C2[0] * xy); DSH(5, SH_C2[1] * yz); DSH(6, SH_C2[2] * (2.f * zz - xx - yy));
                    DSH(7, SH_C2[3] * xz); DSH(8, SH_C2[4] * (xx - yy));
                    for (int c = 0; c < 3; ++c) {
                        dRGBdx[c] += SH_C2[0] * y * SHC(4, c) + SH_C2[2] * 2.f * -x * SHC(6, c) + SH_C2[3] * z * SHC(7, c) + SH_C2[4] * 2.f * x * SHC(8, c);
                        dRGBdy[c] += SH_C2[0] * x * SHC(4, c) + SH_C2[1] * z * SHC(5, c) + SH_C2[2] * 2.f * -y * SHC(6, c) + SH_C2[4] * 2.f * -y * SHC(8, c);
                        dRGBdz[c] += SH_C2[1] * y * SHC(5, c) + SH_C2[2] * 2.f * 2.f * z * SHC(6, c) + SH_C2[3] * x * SHC(7, c);
                    }
                    if (D > 2) {
                        DSH(9, SH_C3[0] * y * (3.f * xx - yy)); DSH(10, SH_C3[1] * xy * z);
                        DSH(11, SH_C3[2] * y * (4.f * zz - xx - yy));
                        DSH(12, SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy));
                        DSH(13, SH_C3[4] * x * (4.f * zz - xx - yy)); DSH(14, SH_C3[5] * z * (xx - yy));
                        DSH(15, SH_C3[6] * x * (xx - 3.f * yy));
                        for (int c = 0; c < 3; ++c) {
                            dRGBdx[c] += (SH_C3[0] * SHC(9, c) * 3.f * 2.f * xy + SH_C3[1] * SHC(10, c) * yz +
                                          SH_C3[2] * SHC(11, c) * -2.f * xy + SH_C3[3] * SHC(12, c) * -3.f * 2.f * xz +
                                          SH_C3[4] * SHC(13, c) * (-3.f * xx + 4.f * zz - yy) +
                                          SH_C3[5] * SHC(14, c) * 2.f * xz + SH_C3[6] * SHC(15, c) * 3.f * (xx - yy));
                            dRGBdy[c] += (SH_C3[0] * SHC(9, c) * 3.f * (xx - yy) + SH_C3[1] * SHC(10, c) * xz +
                                          SH_C3[2] * SHC(11, c) * (-3.f * yy + 4.f * zz - xx) +
                                          SH_C3[3] * SHC(12, c) * -3.f * 2.f * yz + SH_C3[4] * SHC(13, c) * -2.f * xy +
                                          SH_C3[5] * SHC(14, c) * -2.f * yz + SH_C3[6] * SHC(15, c) * -3.f * 2.f * xy);
                            dRGBdz[c] += (SH_C3[1] * SHC(10, c) * xy + SH_C3[2] * SHC(11, c) * 4.f * 2.f * yz +
                                          SH_C3[3] * SHC(12, c) * 3.f * (2.f * zz - xx - yy) +
                                          SH_C3[4] * SHC(13, c) * 4.f * 2.f * xz + SH_C3[5] * SHC(14, c) * (xx - yy));
                        }
                    }
                }
            }
#undef SHC
#undef DSH
            const float ddx = dRGBdx[0] * dRGB[0] + dRGBdx[1] * dRGB[1] + dRGBdx[2] * dRGB[2];
            const float ddy = dRGBdy[0] * dRGB[0] + dRGBdy[1] * dRGB[1] + dRGBdy[2] * dRGB[2];
            const float ddz = dRGBdz[0] * dRGB[0] + dRGBdz[1] * dRGB[1] + dRGBdz[2] * dRGB[2];
            /* dnormvdv: auxiliary.h:105-116 */
            const float sum2 = dox * dox + doy * doy + doz * doz;
            const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
            dmean[0] += ((+sum2 - dox * dox) * ddx - doy * dox * ddy - doz * dox * ddz) * invsum32;
            dmean[1] += (-dox * doy * ddx + (sum2 - doy * doy) * ddy - doz * doy * ddz) * invsum32;
            dmean[2] += (-dox * doz * ddx - doy * doz * ddy + (sum2 - doz * doz) * ddz) * invsum32;
        }
        dL_dmeans[3 * idx] = dmean[0]; dL_dmeans[3 * idx + 1] = dmean[1]; dL_dmeans[3 * idx + 2] = dmean[2];

        if (scales) { /* backward.cu:280-343 */
            const float* q = rotations + 4 * idx;
            const float r = q[0], x = q[1], y = q[2], z = q[3];
            /* glm column-major R: R[c][r] */
            const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                                   {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                                   {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
            const float s[3] = {scale_modifier * scales[3 * idx], scale_modifier * scales[3 * idx + 1],
                                scale_modifier * scales[3 * idx + 2]};
            float Mm[3][3]; /* M = S * R : M[c][r] = S[r][r] * R[c][r] */
            for (int c = 0; c < 3; ++c) for (int rr = 0; rr < 3; ++rr) Mm[c][rr] = s[rr] * R[c][rr];
            const float* d = dcov;
            const float dSig[3][3] = {{d[0], 0.5f * d[1], 0.5f * d[2]}, {0.5f * d[1], d[3], 0.5f * d[4]},
                                      {0.5f * d[2], 0.5f * d[4], d[5]}};
            float dM[3][3]; /* dL_dM = 2 * M * dL_dSigma : (A*B)[c][r] = sum_k A[k][r] * B[c][k] */
            for (int c = 0; c < 3; ++c)
                for (int rr = 0; rr < 3; ++rr)
                    dM[c][rr] = 2.0f * (Mm[0][rr] * dSig[c][0] + Mm[1][rr] * dSig[c][1] + Mm[2][rr] * dSig[c][2]);
            /* Rt = transpose(R): Rt[c][r] = R[r][c]; dL_dMt[c][r] = dM[r][c] */
            float dMt[3][3];
            for (int c = 0; c < 3; ++c) for (int rr = 0; rr < 3; ++rr) dMt[c][rr] = dM[rr][c];
            for (int k = 0; k < 3; ++k)
                dL_dscale[3 * idx + k] = R[0][k] * dMt[k][0] + R[1][k] * dMt[k][1] + R[2][k] * dMt[k][2];
            for (int k = 0; k < 3; ++k) for (int rr = 0; rr < 3; ++rr) dMt[k][rr] *= s[k];
            float* dq = dL_drot + 4 * idx;
            dq[0] = 2 * z * (dMt[0][1] - dMt[1][0]) + 2 * y * (dMt[2][0] - dMt[0][2]) + 2 * x * (dMt[1][2] - dMt[2][1]);
            dq[1] = 2 * y * (dMt[1][0] + dMt[0][1]) + 2 * z * (dMt[2][0] + dMt[0][2]) + 2 * r * (dMt[1][2] - dMt[2][1]) - 4 * x * (dMt[2][2] + dMt[1][1]);
            dq[2] = 2 * x * (dMt[1][0] + dMt[0][1]) + 2 * r * (dMt[2][0] - dMt[0][2]) + 2 * z * (dMt[1][2] + dMt[2][1]) - 4 * y * (dMt[2][2] + dMt[0][0]);
            dq[3] = 2 * r * (dMt[0][1] - dMt[1][0]) + 2 * x * (dMt[2][0] + dMt[0][2]) + 2 * y * (dMt[1][2] + dMt[2][1]) - 4 * z * (dMt[1][1] + dMt[0][0]);
        }
    }
}
