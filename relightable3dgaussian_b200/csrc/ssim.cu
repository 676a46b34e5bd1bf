// Fused SSIM loss: the reference's `ssim(img1, img2)` (utils/loss_utils.py:20-63), called every training step by
// gaussian_renderer/render.py:150 and twice by gaussian_renderer/neilf.py:227,234, as a metric by eval_nvs.py:72 and
// eval_relighting_syn4.py:191,195.  The reference runs five depthwise 11x11 F.conv2d and ~15 elementwise kernels
// forward (and their transposes backward), each moving a full [C,H,W] image through HBM.  Here:
//   forward : ONE tiled kernel (stage x, y with a zero 5-pixel halo; separable 11-tap blur of x, y, x^2, y^2, xy;
//             the SSIM map per pixel; one fp64 partial per CTA) + ONE fixed-order reduction  -> deterministic,
//             and ssim(x, x) is exactly 1 (every factor of the map is bit-identical, the fp64 sum of ones is exact);
//   backward: ONE tiled kernel that recomputes the map terms on a 10-pixel halo and applies the transposed blur
//             (dL/dimg2 is the same kernel with img1 and img2 swapped: the formula is symmetric in IEEE arithmetic).
// All arithmetic is IEEE fp32 (no TF32).  The map's elementwise chain uses explicit intrinsics, so nvcc does not
// contract it into FMAs: every op is rounded on its own, as in the reference's chain of PyTorch kernels.
#include "common.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace r3dg {
namespace {

constexpr int TW = 32, TH = 16;        // output tile of one CTA
constexpr int R = 5;                   // window radius (window_size 11)
constexpr int NT = 256;

// gaussian(11, 1.5) of loss_utils.py:20-22 as the reference rounds it: exp in double, rounded to float32, divided
// by torch's float32 sum.  The reference's 2-D window is the float32-rounded outer product of this vector
// (:26-27); the separable blur applies the exact product, whose entries are <= 0.5 ulp apart from it.  Those
// differences are noise except for their sum: the rounded window weighs 7.0e-9 less in total, and on images with
// dark flat regions (where the map is most sensitive to mu) that DC gain alone moves the mean SSIM by ~2.5e-7,
// 20x the fp32 reference's own error.  The vertical pass therefore adds kGainErr * (centre-row sum), kGainErr =
// sum(window_2d) / sum(w)^2 - 1, to its accumulator before the taps: far below one ulp of any single result, but
// the final rounding is unbiased, so the mean over an image carries the rounded window's gain (the residual is
// ~1e-10 when the two windows are compared in fp64).
__constant__ float kW[11] = {0x1.0d956cp-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f, 0x1.b43c3ep-3f,
                             0x1.106560p-2f,
                             0x1.b43c3ep-3f, 0x1.bff0fep-4f, 0x1.26eb18p-5f, 0x1.f1fe02p-8f, 0x1.0d956cp-10f};
constexpr float kGainErr = -0x1.e41006p-28f;
constexpr float kC1 = static_cast<float>(0.01 * 0.01);
constexpr float kC2 = static_cast<float>(0.03 * 0.03);

// rows x cols window of the plane starting at (gy0, gx0), zero outside the image (F.conv2d's zero padding)
__device__ __forceinline__ void stage(const float* __restrict__ xp, const float* __restrict__ yp, int H, int W, int gy0,
                                      int gx0, int rows, int cols, float* sx, float* sy) {
    for (int i = threadIdx.x; i < rows * cols; i += NT) {
        const int r = i / cols, c = i - r * cols;
        const int gy = gy0 + r, gx = gx0 + c;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        sx[i] = in ? __ldg(xp + (size_t)gy * W + gx) : 0.0f;
        sy[i] = in ? __ldg(yp + (size_t)gy * W + gx) : 0.0f;
    }
}

// horizontal 11-tap pass of x, y, x*x, y*y, x*y: `rows` rows of width `ow` into h[5][rows][ow] (input stride ow + 2R)
__device__ __forceinline__ void hblur5(const float* sx, const float* sy, int rows, int ow, float* h) {
    const int iw = ow + 2 * R, n = rows * ow;
    for (int i = threadIdx.x; i < n; i += NT) {
        const int r = i / ow, c = i - r * ow;
        const float* px = sx + r * iw + c;
        const float* py = sy + r * iw + c;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
#pragma unroll
        for (int k = 0; k < 2 * R + 1; ++k) {
            const float xv = px[k], yv = py[k], w = kW[k];
            a0 = fma_(w, xv, a0);
            a1 = fma_(w, yv, a1);
            a2 = fma_(w, mul_(xv, xv), a2);          // img1 * img1 is its own rounded tensor in the reference
            a3 = fma_(w, mul_(yv, yv), a3);
            a4 = fma_(w, mul_(xv, yv), a4);
        }
        h[i] = a0; h[n + i] = a1; h[2 * n + i] = a2; h[3 * n + i] = a3; h[4 * n + i] = a4;
    }
}

// vertical 11-tap pass at (r, c) of the five planes h[5][rows][ow], with the window's gain correction (above)
__device__ __forceinline__ void vblur5(const float* h, int rows, int ow, int r, int c, float* q) {
    const int n = rows * ow, jc = (r + R) * ow + c;
    float a0 = mul_(kGainErr, h[jc]), a1 = mul_(kGainErr, h[n + jc]), a2 = mul_(kGainErr, h[2 * n + jc]),
          a3 = mul_(kGainErr, h[3 * n + jc]), a4 = mul_(kGainErr, h[4 * n + jc]);
#pragma unroll
    for (int k = 0; k < 2 * R + 1; ++k) {
        const int j = (r + k) * ow + c;
        const float w = kW[k];
        a0 = fma_(w, h[j], a0);
        a1 = fma_(w, h[n + j], a1);
        a2 = fma_(w, h[2 * n + j], a2);
        a3 = fma_(w, h[3 * n + j], a3);
        a4 = fma_(w, h[4 * n + j], a4);
    }
    q[0] = a0; q[1] = a1; q[2] = a2; q[3] = a3; q[4] = a4;
}

struct MapTerms {
    float mu1, mu2, A, B, Cc, D, m;
};

// loss_utils.py:47-58 op for op: q = {mu1, mu2, G*(x*x), G*(y*y), G*(x*y)}
__device__ __forceinline__ MapTerms ssim_map(const float* q) {
    MapTerms t;
    t.mu1 = q[0]; t.mu2 = q[1];
    const float mu1_sq = mul_(t.mu1, t.mu1), mu2_sq = mul_(t.mu2, t.mu2), mu1_mu2 = mul_(t.mu1, t.mu2);
    const float s11 = sub_(q[2], mu1_sq), s22 = sub_(q[3], mu2_sq), s12 = sub_(q[4], mu1_mu2);
    t.A = add_(mul_(2.0f, mu1_mu2), kC1);
    t.B = add_(mul_(2.0f, s12), kC2);
    t.Cc = add_(add_(mu1_sq, mu2_sq), kC1);
    t.D = add_(add_(s11, s22), kC2);
    t.m = div_(mul_(t.A, t.B), mul_(t.Cc, t.D));
    return t;
}

__global__ void __launch_bounds__(NT) ssim_fwd_kernel(int H, int W, const float* __restrict__ x, const float* __restrict__ y,
                                                      double* __restrict__ partial) {
    constexpr int SR = TH + 2 * R, SC = TW + 2 * R;
    __shared__ float sx[SR * SC], sy[SR * SC];
    __shared__ float h[5 * SR * TW];
    const size_t plane = (size_t)blockIdx.z * H * W;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    stage(x + plane, y + plane, H, W, y0 - R, x0 - R, SR, SC, sx, sy);
    __syncthreads();
    hblur5(sx, sy, SR, TW, h);
    __syncthreads();
    double acc = 0.0;
    for (int i = threadIdx.x; i < TH * TW; i += NT) {
        const int r = i / TW, c = i - r * TW;
        if (y0 + r < H && x0 + c < W) {
            float q[5];
            vblur5(h, SR, TW, r, c, q);
            acc += (double)ssim_map(q).m;
        }
    }
    cta_partial<NT>(acc, partial + ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x);
}

// dL/dx = s * (G*alpha + 2x (G*beta) + y (G*gamma)) over in-image pixels, with the map terms
//   beta = dm/ds11 = -m/D,  gamma = dm/ds12 = 2A/(Cc D),  alpha = dm/dmu1 - 2 mu1 beta - mu2 gamma
// recomputed on the tile plus a 5-pixel halo (zero outside the image: the transposed blur of a zero-padded blur),
// from x, y staged with a 10-pixel halo.  G is symmetric, so its transpose is the same blur.
__global__ void __launch_bounds__(NT) ssim_bwd_kernel(int C, int H, int W, const float* __restrict__ x,
                                                      const float* __restrict__ y, const float* __restrict__ g,
                                                      int g_per_image, float count, float* __restrict__ dx) {
    constexpr int IR = TH + 4 * R, IC = TW + 4 * R;       // staged x, y
    constexpr int MR = TH + 2 * R, MC = TW + 2 * R;       // map terms
    __shared__ float s_in[2 * IR * IC];                   // x | y, then alpha | beta | gamma [3][MR][MC]
    __shared__ float s_h[5 * IR * MC];                    // horizontal sums of the 5 blurs, then of the 3 terms [3][MR][TW]
    static_assert(3 * MR * MC <= 2 * IR * IC && 3 * MR * TW <= 5 * IR * MC, "aliased buffers");
    const size_t plane = (size_t)blockIdx.z * H * W;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const float* xp = x + plane;
    const float* yp = y + plane;
    stage(xp, yp, H, W, y0 - 2 * R, x0 - 2 * R, IR, IC, s_in, s_in + IR * IC);
    __syncthreads();
    hblur5(s_in, s_in + IR * IC, IR, MC, s_h);
    __syncthreads();
    constexpr int MN = MR * MC;
    for (int i = threadIdx.x; i < MN; i += NT) {
        const int r = i / MC, c = i - r * MC;
        const int gy = y0 - R + r, gx = x0 - R + c;
        float alpha = 0.f, beta = 0.f, gamma = 0.f;
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
            float q[5];
            vblur5(s_h, IR, MC, r, c, q);
            const MapTerms t = ssim_map(q);
            const float CD = t.Cc * t.D;
            beta = -t.m / t.D;
            gamma = 2.0f * t.A / CD;
            const float dmu1 = 2.0f * t.mu2 * t.B / CD - 2.0f * t.mu1 * t.m / t.Cc;
            alpha = dmu1 - 2.0f * t.mu1 * beta - t.mu2 * gamma;
        }
        s_in[i] = alpha; s_in[MN + i] = beta; s_in[2 * MN + i] = gamma;
    }
    __syncthreads();
    constexpr int HN = MR * TW;
    for (int i = threadIdx.x; i < HN; i += NT) {
        const int r = i / TW, c = i - r * TW;
        const float* p = s_in + r * MC + c;
        float a = 0.f, b = 0.f, e = 0.f;
#pragma unroll
        for (int k = 0; k < 2 * R + 1; ++k) {
            a = fmaf(kW[k], p[k], a);
            b = fmaf(kW[k], p[MN + k], b);
            e = fmaf(kW[k], p[2 * MN + k], e);
        }
        s_h[i] = a; s_h[HN + i] = b; s_h[2 * HN + i] = e;
    }
    __syncthreads();
    const float s = g[g_per_image ? blockIdx.z / C : 0] / count;
    for (int i = threadIdx.x; i < TH * TW; i += NT) {
        const int r = i / TW, c = i - r * TW;
        const int gy = y0 + r, gx = x0 + c;
        if (gy >= H || gx >= W) continue;
        float a = 0.f, b = 0.f, e = 0.f;
#pragma unroll
        for (int k = 0; k < 2 * R + 1; ++k) {
            const int j = (r + k) * TW + c;
            a = fmaf(kW[k], s_h[j], a);
            b = fmaf(kW[k], s_h[HN + j], b);
            e = fmaf(kW[k], s_h[2 * HN + j], e);
        }
        const size_t o = (size_t)gy * W + gx;
        dx[plane + o] = s * (a + 2.0f * __ldg(xp + o) * b + __ldg(yp + o) * e);
    }
}

int check_shape(int N, int C, int H, int W) {
    if (N <= 0 || C <= 0 || H <= 0 || W <= 0) return R3DG_ERR_BAD_ARG;
    if ((long long)N * C > 65535 || (long long)H * W > (1LL << 31) - 1 || (H + TH - 1) / TH > 65535)
        return R3DG_ERR_UNSUPPORTED;                     // grid.z = planes, grid.y = tile rows, int pixel offsets
    return 0;
}

dim3 tile_grid(int N, int C, int H, int W) { return dim3((W + TW - 1) / TW, (H + TH - 1) / TH, N * C); }

}  // namespace

size_t ssim_tmp_bytes(int N, int C, int H, int W) {
    if (check_shape(N, C, H, W) != 0) return 0;
    const dim3 gr = tile_grid(N, C, H, W);
    return ((size_t)gr.x * gr.y * gr.z * sizeof(double) + 255) & ~(size_t)255;
}

int launch_ssim_forward(int N, int C, int H, int W, const float* img1, const float* img2, int size_average, float* out,
                        void* tmp, size_t tmp_bytes, cudaStream_t stream) {
    const int rc = check_shape(N, C, H, W);
    if (rc != 0) return rc;
    if (!img1 || !img2 || !out || !tmp || tmp_bytes < ssim_tmp_bytes(N, C, H, W)) return R3DG_ERR_BAD_ARG;
    const dim3 gr = tile_grid(N, C, H, W);
    double* partial = (double*)tmp;
    ssim_fwd_kernel<<<gr, NT, 0, stream>>>(H, W, img1, img2, partial);
    R3DG_CUDA_TRY(cudaGetLastError());
    const long long per_image = (long long)gr.x * gr.y * C;
    const int outs = size_average ? 1 : N;
    const double count = (double)C * H * W * (size_average ? N : 1);
    reduce_partials_kernel<<<outs, kReduceNT, 0, stream>>>(partial, per_image * N / outs, count, out);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_ssim_backward(int N, int C, int H, int W, const float* img1, const float* img2, int size_average,
                         const float* dL_dout, float* dL_dimg1, cudaStream_t stream) {
    const int rc = check_shape(N, C, H, W);
    if (rc != 0) return rc;
    if (!img1 || !img2 || !dL_dout || !dL_dimg1) return R3DG_ERR_BAD_ARG;
    const float count = (float)((double)C * H * W * (size_average ? N : 1));
    ssim_bwd_kernel<<<tile_grid(N, C, H, W), NT, 0, stream>>>(C, H, W, img1, img2, dL_dout, size_average ? 0 : 1, count,
                                                              dL_dimg1);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
