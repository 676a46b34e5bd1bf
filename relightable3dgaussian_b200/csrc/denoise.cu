// G-buffer-guided a-trous denoiser (include/r3dg_b200.h, DENOISE; DESIGN.md §4.32): L passes of a 5 x 5 cross-bilateral
// stencil at steps 1, 2, 4, ... whose weights come from the normal, point, mask and feature guides only, so the filter is
// linear in the image and its backward is the transposed stencil.  Compiled with -fmad=false: the forward and the
// backward evaluate every weight with the same function on the same records, and without FMA contraction the two
// kernels round it alike, so each backward weight is the forward's bit for bit.
//
// Design notes
//  * a pack kernel writes each pixel's guides once per call as float4 planes: (n^, valid), (point, f_0) and, for
//    F > 1, (f_1..f_4) and (f_5..f_7, 0).  Feature slots past F hold 0 in every pixel, so they add exactly +0 to
//    |f_p - f_q|^2 and every pass reads whole planes without a per-feature branch.
//  * one thread per pixel, 32 x 8 pixel CTAs and one grid z per view: a warp's taps at any step are 32 consecutive
//    pixels of one row, so every record and image load is coalesced and the step-1 and step-2 taps hit L1.
//  * forward: acc = sum_o w x and W = sum_o w in tap order, y = acc * (1 / W), 1 / W stored per pass.  Backward: the
//    gather g_k(q) = sum_o w(q - s o, q) (g(q - s o) (1 / W(q - s o))) in the same tap order: no atomics.
//  * invalid taps are skipped before their image values are read, so a masked pixel's x (NaN included) is never used.
#include <cmath>

#include "kernels.h"

namespace r3dg {

#define DN_BX 32
#define DN_BY 8
#define DN_LOG2E 1.4426950408889634f

struct DenoisePass {
    const float4* rec;          // NR planes of npix float4
    size_t npix;                // V H W
    int H, W, C, step;
    float sigma_normal, inv_plane, inv_features2;
    const float* src;           // [V,C,H,W]
    float* dst;                 // [V,C,H,W]
    float* inv_w;               // [V,H,W] of this pass: written by the forward, read by the backward
};

__constant__ float c_dn_h[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};

template <int NR>
__device__ __forceinline__ void load_record(const DenoisePass& p, int pix, float4 (&r)[NR]) {
#pragma unroll
    for (int i = 0; i < NR; ++i) r[i] = __ldg(p.rec + (size_t)i * p.npix + pix);
}

// w(p, q) of a tap q != p with filter weight hh = h(o_x) h(o_y): the one weight function of both directions
template <int NR>
__device__ __forceinline__ float tap_weight(const DenoisePass& p, const float4 (&rp)[NR], const float4 (&rq)[NR], float hh) {
    const float c = fminf(fmaxf(rp[0].x * rq[0].x + rp[0].y * rq[0].y + rp[0].z * rq[0].z, 0.f), 1.f);
    const float dx = rq[1].x - rp[1].x, dy = rq[1].y - rp[1].y, dz = rq[1].z - rp[1].z;
    const float dd = dx * dx + dy * dy + dz * dz;
    const float t = dd > 0.f ? fabsf(rp[0].x * dx + rp[0].y * dy + rp[0].z * dz) / sqrtf(dd) : 0.f;
    float df = rq[1].w - rp[1].w;
    float f2 = df * df;
#pragma unroll
    for (int i = 2; i < NR; ++i) {
        df = rq[i].x - rp[i].x; f2 = f2 + df * df;
        df = rq[i].y - rp[i].y; f2 = f2 + df * df;
        df = rq[i].z - rp[i].z; f2 = f2 + df * df;
        df = rq[i].w - rp[i].w; f2 = f2 + df * df;
    }
    const float e = p.sigma_normal * log2f(c) - (t * p.inv_plane + f2 * p.inv_features2) * DN_LOG2E;
    return hh * exp2f(e);
}

// the guides of every pixel as NR float4 planes; invalid pixels get an all-zero record
__global__ void __launch_bounds__(256) denoise_pack_kernel(const r3dg_denoise_args a, float4* rec, int NR, size_t npix) {
    const size_t HW = (size_t)a.H * a.W;
    for (size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += (size_t)gridDim.x * blockDim.x) {
        const size_t v = pix / HW, q = pix - v * HW;
        float4 r[4] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f),
                       make_float4(0.f, 0.f, 0.f, 0.f)};
        if (!a.mask || a.mask[pix]) {
            const float* n = a.normal + 3 * v * HW + q;
            const float* x = a.points + 3 * v * HW + q;
            const float nx = n[0], ny = n[HW], nz = n[2 * HW];
            const float len = fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-12f);
            r[0] = make_float4(nx / len, ny / len, nz / len, 1.f);
            float f[R3DG_DENOISE_MAX_FEATURES + 1];
#pragma unroll
            for (int j = 0; j <= R3DG_DENOISE_MAX_FEATURES; ++j)
                f[j] = j < a.F ? a.features[((size_t)a.F * v + j) * HW + q] : 0.f;
            r[1] = make_float4(x[0], x[HW], x[2 * HW], f[0]);
            r[2] = make_float4(f[1], f[2], f[3], f[4]);
            r[3] = make_float4(f[5], f[6], f[7], f[8]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (i < NR) rec[i * npix + pix] = r[i];
    }
}

__device__ __forceinline__ bool pixel_of_thread(const DenoisePass& p, int& x, int& y, int& v) {
    x = blockIdx.x * DN_BX + threadIdx.x;
    y = blockIdx.y * DN_BY + threadIdx.y;
    v = blockIdx.z;
    return x < p.W && y < p.H;
}

// one forward pass: dst = the stencil of src, and 1 / W
template <int NR>
__global__ void __launch_bounds__(DN_BX * DN_BY, 3) denoise_fwd_kernel(const DenoisePass p) {
    int x, y, v;
    if (!pixel_of_thread(p, x, y, v)) return;
    const int HW = p.H * p.W, yx = y * p.W + x, pix = v * HW + yx;
    const float* src = p.src + v * p.C * HW;
    float* dst = p.dst + v * p.C * HW + yx;
    float4 rp[NR];
    load_record<NR>(p, pix, rp);
    if (rp[0].w == 0.f) {
        for (int c = 0; c < p.C; ++c) dst[c * HW] = 0.f;
        p.inv_w[pix] = 0.f;
        return;
    }
    float acc[R3DG_DENOISE_MAX_CHANNELS], wsum = 0.f;
#pragma unroll
    for (int c = 0; c < R3DG_DENOISE_MAX_CHANNELS; ++c) acc[c] = 0.f;
    for (int oy = -2; oy <= 2; ++oy) {
        const int qy = y + oy * p.step;
        if (qy < 0 || qy >= p.H) continue;
        for (int ox = -2; ox <= 2; ++ox) {
            const int qx = x + ox * p.step;
            if (qx < 0 || qx >= p.W) continue;
            const int qyx = qy * p.W + qx;
            float w;
            if (oy == 0 && ox == 0) {
                w = 0.140625f;                                         // h(0)^2
            } else {
                float4 rq[NR];
                load_record<NR>(p, v * HW + qyx, rq);
                if (rq[0].w == 0.f) continue;
                w = tap_weight<NR>(p, rp, rq, c_dn_h[oy + 2] * c_dn_h[ox + 2]);
            }
            wsum = wsum + w;
#pragma unroll
            for (int c = 0; c < R3DG_DENOISE_MAX_CHANNELS; ++c)
                if (c < p.C) acc[c] = acc[c] + w * __ldg(src + c * HW + qyx);
        }
    }
    const float inv = 1.f / wsum;
    p.inv_w[pix] = inv;
#pragma unroll
    for (int c = 0; c < R3DG_DENOISE_MAX_CHANNELS; ++c)
        if (c < p.C) dst[c * HW] = acc[c] * inv;
}

// one backward pass: dst(q) = sum_o w(q - s o, q) src(q - s o) / W(q - s o)
template <int NR>
__global__ void __launch_bounds__(DN_BX * DN_BY, 3) denoise_bwd_kernel(const DenoisePass p) {
    int x, y, v;
    if (!pixel_of_thread(p, x, y, v)) return;
    const int HW = p.H * p.W, yx = y * p.W + x, pix = v * HW + yx;
    const float* src = p.src + v * p.C * HW;
    float* dst = p.dst + v * p.C * HW + yx;
    float4 rq[NR];
    load_record<NR>(p, pix, rq);
    if (rq[0].w == 0.f) {
        for (int c = 0; c < p.C; ++c) dst[c * HW] = 0.f;
        return;
    }
    const float* inv_w = p.inv_w + v * HW;
    float acc[R3DG_DENOISE_MAX_CHANNELS];
#pragma unroll
    for (int c = 0; c < R3DG_DENOISE_MAX_CHANNELS; ++c) acc[c] = 0.f;
    for (int oy = -2; oy <= 2; ++oy) {
        const int py = y - oy * p.step;
        if (py < 0 || py >= p.H) continue;
        for (int ox = -2; ox <= 2; ++ox) {
            const int px = x - ox * p.step;
            if (px < 0 || px >= p.W) continue;
            const int pyx = py * p.W + px;
            float w;
            if (oy == 0 && ox == 0) {
                w = 0.140625f;
            } else {
                float4 rp[NR];
                load_record<NR>(p, v * HW + pyx, rp);
                if (rp[0].w == 0.f) continue;
                w = tap_weight<NR>(p, rp, rq, c_dn_h[oy + 2] * c_dn_h[ox + 2]);
            }
            const float inv = __ldg(inv_w + pyx);
#pragma unroll
            for (int c = 0; c < R3DG_DENOISE_MAX_CHANNELS; ++c)
                if (c < p.C) acc[c] = acc[c] + w * (__ldg(src + c * HW + pyx) * inv);
        }
    }
#pragma unroll
    for (int c = 0; c < R3DG_DENOISE_MAX_CHANNELS; ++c)
        if (c < p.C) dst[c * HW] = acc[c];
}

static int denoise_planes(int F) { return F <= 1 ? 2 : 2 + (F + 2) / 4; }

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// the workspace regions: records, 1 / W of the L passes, the ping-pong image
struct DenoiseWork {
    float4* rec;
    float* inv_w;
    float* tmp;
};

static DenoiseWork denoise_work(const r3dg_denoise_args* a) {
    const size_t npix = (size_t)a->V * a->H * a->W;
    char* w = (char*)a->work;
    DenoiseWork d;
    d.rec = (float4*)w;
    w += align256((size_t)denoise_planes(a->F) * npix * sizeof(float4));
    d.inv_w = (float*)w;
    w += align256((size_t)a->L * npix * sizeof(float));
    d.tmp = (float*)w;
    return d;
}

// the checks of both directions: 0, or the call's R3DG_ERR_* code
static int denoise_check(const r3dg_denoise_args* a) {
    if (!a || a->V < 1 || a->V > R3DG_MAX_VIEWS || a->H < 1 || a->W < 1 || a->C < 1 || a->C > R3DG_DENOISE_MAX_CHANNELS ||
        a->F < 0 || a->F > R3DG_DENOISE_MAX_FEATURES || a->L < 1 || a->L > R3DG_DENOISE_MAX_PASSES)
        return R3DG_ERR_BAD_ARG;
    const float sigmas[3] = {a->sigma_normal, a->sigma_plane, a->sigma_features};
    for (const float s : sigmas)
        if (!(s > 0.f) || !std::isfinite(s)) return R3DG_ERR_BAD_ARG;
    const size_t need = r3dg_denoise_work_bytes(a->V, a->H, a->W, a->C, a->F, a->L);
    if (!a->work || a->work_bytes < need) return R3DG_ERR_BAD_ARG;
    const long long wide = a->C > a->F ? a->C : a->F;
    if ((long long)a->V * a->H * a->W * wide >= (1LL << 31)) return R3DG_ERR_UNSUPPORTED;
    return 0;
}

static DenoisePass denoise_pass(const r3dg_denoise_args* a, const DenoiseWork& d, int k) {
    DenoisePass p;
    p.rec = d.rec;
    p.npix = (size_t)a->V * a->H * a->W;
    p.H = a->H; p.W = a->W; p.C = a->C; p.step = 1 << k;
    p.sigma_normal = a->sigma_normal;
    p.inv_plane = 1.f / a->sigma_plane;
    p.inv_features2 = 1.f / (a->sigma_features * a->sigma_features);
    p.inv_w = d.inv_w + (size_t)k * p.npix;
    return p;
}

template <int NR>
static void launch_pass(bool forward, const DenoisePass& p, int V, cudaStream_t stream) {
    const dim3 grid((p.W + DN_BX - 1) / DN_BX, (p.H + DN_BY - 1) / DN_BY, V), block(DN_BX, DN_BY);
    if (forward) denoise_fwd_kernel<NR><<<grid, block, 0, stream>>>(p);
    else denoise_bwd_kernel<NR><<<grid, block, 0, stream>>>(p);
}

static void launch_pass(bool forward, int NR, const DenoisePass& p, int V, cudaStream_t stream) {
    if (NR == 2) launch_pass<2>(forward, p, V, stream);
    else if (NR == 3) launch_pass<3>(forward, p, V, stream);
    else launch_pass<4>(forward, p, V, stream);
}

}  // namespace r3dg

// ---- C ABI --------------------------------------------------------------------------------------
using namespace r3dg;
extern "C" {

size_t r3dg_denoise_work_bytes(int V, int H, int W, int C, int F, int L) {
    if (V < 1 || H < 1 || W < 1 || C < 1 || F < 0 || L < 1) return 0;
    const size_t npix = (size_t)V * H * W;
    return align256((size_t)denoise_planes(F) * npix * sizeof(float4)) + align256((size_t)L * npix * sizeof(float)) +
           align256((size_t)C * npix * sizeof(float));
}

int r3dg_denoise_forward(const r3dg_denoise_args* a, r3dg_stream_t stream_) {
    const int err = denoise_check(a);
    if (err != 0) return err;
    if (!a->normal || !a->points || (a->F > 0 && !a->features) || !a->x || !a->y) return R3DG_ERR_BAD_ARG;
    const cudaStream_t stream = (cudaStream_t)stream_;
    const DenoiseWork d = denoise_work(a);
    const int NR = denoise_planes(a->F);
    const size_t npix = (size_t)a->V * a->H * a->W;
    const int blocks = (int)((npix + 255) / 256 < 8192 ? (npix + 255) / 256 : 8192);
    denoise_pack_kernel<<<blocks, 256, 0, stream>>>(*a, d.rec, NR, npix);
    R3DG_CUDA_TRY(cudaGetLastError());
    // pass k writes y when L - 1 - k is even, else tmp: the last pass writes y and no pass reads what it writes
    for (int k = 0; k < a->L; ++k) {
        DenoisePass p = denoise_pass(a, d, k);
        p.src = k == 0 ? a->x : ((a->L - k) % 2 == 0 ? a->y : d.tmp);
        p.dst = (a->L - 1 - k) % 2 == 0 ? a->y : d.tmp;
        launch_pass(true, NR, p, a->V, stream);
        R3DG_CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

int r3dg_denoise_backward(const r3dg_denoise_args* a, r3dg_stream_t stream_) {
    const int err = denoise_check(a);
    if (err != 0) return err;
    if (!a->dL_dy || !a->dL_dx) return R3DG_ERR_BAD_ARG;
    const cudaStream_t stream = (cudaStream_t)stream_;
    const DenoiseWork d = denoise_work(a);
    const int NR = denoise_planes(a->F);
    // pass k (from L - 1 down to 0) writes dL_dx when k is even, else tmp: pass 0 writes dL_dx
    for (int k = a->L - 1; k >= 0; --k) {
        DenoisePass p = denoise_pass(a, d, k);
        p.src = k == a->L - 1 ? a->dL_dy : ((k + 1) % 2 == 0 ? a->dL_dx : d.tmp);
        p.dst = k % 2 == 0 ? a->dL_dx : d.tmp;
        launch_pass(false, NR, p, a->V, stream);
        R3DG_CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

}  // extern "C"
