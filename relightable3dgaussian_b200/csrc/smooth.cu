// Fused smoothness regularisers of the reference's training loss (utils/loss_utils.py:104-105,113-117):
//   first_order_edge_aware_loss(data, img) = mean over (c, y, x) of sum_d |S_d(D_c)| * exp(-|S_d(I_c)|), where S_x,
//     S_y are kornia's normalised Sobel responses (kernel / 8, replicate padding of 1) and a 1-channel input is
//     broadcast over the channels of the other.  Called by gaussian_renderer/render.py:170 and three times per step
//     by gaussian_renderer/neilf.py:284,291,299; the reference runs two spatial_gradient convolutions and ~a dozen
//     elementwise kernels forward, more backward.
//   tv_loss(x) = mean of the squared vertical differences + mean of the squared horizontal ones
//     (gaussian_renderer/neilf.py:306,312).
// Here each is ONE tiled forward kernel writing an fp64 partial per CTA + the shared fixed-order reduction
// (reduce.cuh), and ONE backward kernel in gather form: every thread owns input pixels and collects from the output
// pixels that read them (for the edge-aware loss, including the taps that replicate padding folds onto the border).
// No float atomics, so values and gradients are bit-reproducible run to run.  IEEE fp32 throughout (the reference's
// convolutions run in TF32 under torch's defaults); expf, no flush-to-zero.
#include "common.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace r3dg {
namespace {

constexpr int TW = 32, TH = 16;        // pixel tile of one CTA
constexpr int NT = 256;
constexpr int PPT = TW * TH / NT;      // pixels per thread in the backward gather

// rows x cols window of the plane starting at (gy0, gx0), indices clamped to the image (replicate padding)
__device__ __forceinline__ void stage_clamped(const float* __restrict__ p, int H, int W, int gy0, int gx0, int rows,
                                              int cols, float* s) {
    for (int i = threadIdx.x; i < rows * cols; i += NT) {
        const int r = i / cols, c = i - r * cols;
        const int gy = min(max(gy0 + r, 0), H - 1), gx = min(max(gx0 + c, 0), W - 1);
        s[i] = __ldg(p + (size_t)gy * W + gx);
    }
}

// Normalised Sobel responses at s[k] (row stride ld), written as differences of opposite taps, so a constant
// neighbourhood gives exactly 0 (as the reference's convolution does).  * 0.125 is the exact / 8.
__device__ __forceinline__ float sobel_x(const float* s, int k, int ld) {
    const float t = sub_(s[k - ld + 1], s[k - ld - 1]), m = sub_(s[k + 1], s[k - 1]), b = sub_(s[k + ld + 1], s[k + ld - 1]);
    return mul_(add_(add_(t, mul_(2.0f, m)), b), 0.125f);
}
__device__ __forceinline__ float sobel_y(const float* s, int k, int ld) {
    const float l = sub_(s[k + ld - 1], s[k - ld - 1]), m = sub_(s[k + ld], s[k - ld]), r = sub_(s[k + ld + 1], s[k - ld + 1]);
    return mul_(add_(add_(l, mul_(2.0f, m)), r), 0.125f);
}

// torch.sign, the derivative torch's abs backward uses: 0 at 0, so pixels where a response is exactly 0 (masked or
// flat regions) pass no gradient
__device__ __forceinline__ float sign0(float v) { return v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : 0.0f); }

// Transposed stencils at padded position k of the output-gradient maps gx (of S_x) and gy (of S_y), row stride ld:
// sum over taps t of w_t * G[k - t].  The maps are 0 outside the image, where there are no output pixels.
__device__ __forceinline__ float sobel_adjoint(const float* gx, const float* gy, int k, int ld) {
    const float ax = add_(add_(sub_(gx[k + ld - 1], gx[k + ld + 1]), mul_(2.0f, sub_(gx[k - 1], gx[k + 1]))),
                          sub_(gx[k - ld - 1], gx[k - ld + 1]));
    const float ay = add_(add_(sub_(gy[k - ld + 1], gy[k + ld + 1]), mul_(2.0f, sub_(gy[k - ld], gy[k + ld]))),
                          sub_(gy[k - ld - 1], gy[k + ld - 1]));
    return mul_(add_(ax, ay), 0.125f);
}

// One CTA per TW x TH tile of output channel blockIdx.z; a 1-channel input supplies its only plane to every channel.
__global__ void __launch_bounds__(NT) edge_fwd_kernel(int Cd, int Ci, int H, int W, const float* __restrict__ data,
                                                      const float* __restrict__ img, double* __restrict__ partial) {
    constexpr int SR = TH + 2, SC = TW + 2;
    __shared__ float sd[SR * SC], si[SR * SC];
    const size_t HW = (size_t)H * W;
    const int c = blockIdx.z, x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    stage_clamped(data + (Cd > 1 ? c : 0) * HW, H, W, y0 - 1, x0 - 1, SR, SC, sd);
    stage_clamped(img + (Ci > 1 ? c : 0) * HW, H, W, y0 - 1, x0 - 1, SR, SC, si);
    __syncthreads();
    double acc = 0.0;
    for (int i = threadIdx.x; i < TH * TW; i += NT) {
        const int r = i / TW, cc = i - r * TW;
        if (y0 + r < H && x0 + cc < W) {
            const int k = (r + 1) * SC + cc + 1;
            const float px = mul_(fabsf(sobel_x(sd, k, SC)), expf(-fabsf(sobel_x(si, k, SC))));
            const float py = mul_(fabsf(sobel_y(sd, k, SC)), expf(-fabsf(sobel_y(si, k, SC))));
            acc += (double)add_(px, py);                 // .sum(1) over the two directions, in fp32
        }
    }
    cta_partial<NT>(acc, partial + ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x);
}

// dL/ddata and / or dL/dimg (either may be NULL) for the input pixels of one TW x TH tile.  Per channel: the output
// gradients of the four responses (torch's abs / exp / mul backward) on the tile plus a 2-pixel halo, then for each
// input pixel the transposed stencil at the padded positions that replicate onto it: itself, and at the image border
// the pad row / column (and corner) beyond it.  With Cd == Ci a CTA does channel blockIdx.z; otherwise it loops over
// all C channels, summing the 1-channel input's gradient in registers and writing the other's plane by plane.
__global__ void __launch_bounds__(NT) edge_bwd_kernel(int C, int Cd, int Ci, int H, int W, const float* __restrict__ data,
                                                      const float* __restrict__ img, const float* __restrict__ g,
                                                      float count, float* __restrict__ dD, float* __restrict__ dI) {
    constexpr int GR = TH + 4, GC = TW + 4;          // output gradients
    constexpr int SR = GR + 2, SC = GC + 2;          // staged inputs
    constexpr int GN = GR * GC;
    __shared__ float sd[SR * SC], si[SR * SC];
    __shared__ float gm[4 * GN];                     // d/dS_x(D), d/dS_y(D), d/dS_x(I), d/dS_y(I)
    const size_t HW = (size_t)H * W;
    const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const int c0 = Cd == Ci ? (int)blockIdx.z : 0, c1 = Cd == Ci ? c0 + 1 : C;
    const float s = div_(g[0], count);               // mean backward
    float accD[PPT], accI[PPT];
#pragma unroll
    for (int j = 0; j < PPT; ++j) accD[j] = accI[j] = 0.0f;
    for (int c = c0; c < c1; ++c) {
        if (c > c0) __syncthreads();                 // the previous channel's gather is done with the buffers
        stage_clamped(data + (Cd > 1 ? c : 0) * HW, H, W, y0 - 3, x0 - 3, SR, SC, sd);
        stage_clamped(img + (Ci > 1 ? c : 0) * HW, H, W, y0 - 3, x0 - 3, SR, SC, si);
        __syncthreads();
        for (int i = threadIdx.x; i < GN; i += NT) {
            const int r = i / GC, cc = i - r * GC;
            const int gy = y0 - 2 + r, gx = x0 - 2 + cc;
            float gdx = 0.f, gdy = 0.f, gix = 0.f, giy = 0.f;
            if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
                const int k = (r + 1) * SC + cc + 1;
                const float dx = sobel_x(sd, k, SC), dy = sobel_y(sd, k, SC);
                const float ix = sobel_x(si, k, SC), iy = sobel_y(si, k, SC);
                const float ex = expf(-fabsf(ix)), ey = expf(-fabsf(iy));
                gdx = mul_(mul_(s, ex), sign0(dx));
                gdy = mul_(mul_(s, ey), sign0(dy));
                gix = mul_(-mul_(mul_(s, fabsf(dx)), ex), sign0(ix));
                giy = mul_(-mul_(mul_(s, fabsf(dy)), ey), sign0(iy));
            }
            gm[i] = gdx; gm[GN + i] = gdy; gm[2 * GN + i] = gix; gm[3 * GN + i] = giy;
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < PPT; ++j) {
            const int i = threadIdx.x + j * NT;
            const int r = i / TW, cc = i - r * TW;
            const int gy = y0 + r, gx = x0 + cc;
            if (gy >= H || gx >= W) continue;
            const int k = (r + 2) * GC + cc + 2;
            const int uy0 = gy == 0 ? -1 : 0, uy1 = gy == H - 1 ? 1 : 0;
            const int ux0 = gx == 0 ? -1 : 0, ux1 = gx == W - 1 ? 1 : 0;
            float vD = 0.f, vI = 0.f;
            for (int uy = uy0; uy <= uy1; ++uy)
                for (int ux = ux0; ux <= ux1; ++ux) {
                    const int ku = k + uy * GC + ux;
                    if (dD) vD = add_(vD, sobel_adjoint(gm, gm + GN, ku, GC));
                    if (dI) vI = add_(vI, sobel_adjoint(gm + 2 * GN, gm + 3 * GN, ku, GC));
                }
            accD[j] = add_(accD[j], vD);
            accI[j] = add_(accI[j], vI);
        }
        const bool lastc = c + 1 == c1;
#pragma unroll
        for (int j = 0; j < PPT; ++j) {
            const int i = threadIdx.x + j * NT;
            const int r = i / TW, cc = i - r * TW;
            const int gy = y0 + r, gx = x0 + cc;
            if (gy >= H || gx >= W) continue;
            const size_t o = (size_t)gy * W + gx;
            if (dD && (Cd > 1 || lastc)) { dD[(Cd > 1 ? c : 0) * HW + o] = accD[j]; accD[j] = 0.0f; }
            if (dI && (Ci > 1 || lastc)) { dI[(Ci > 1 ? c : 0) * HW + o] = accI[j]; accI[j] = 0.0f; }
        }
    }
}

int check_edge(int Cd, int Ci, int H, int W) {
    if (Cd <= 0 || Ci <= 0 || H <= 0 || W <= 0) return R3DG_ERR_BAD_ARG;
    const int C = max(Cd, Ci);
    if ((Cd != 1 && Cd != C) || (Ci != 1 && Ci != C)) return R3DG_ERR_BAD_ARG;    // torch broadcasting raises too
    if (C > 65535 || (long long)H * W > (1LL << 31) - 1 || (H + TH - 1) / TH > 65535)
        return R3DG_ERR_UNSUPPORTED;                     // grid.z = channels, grid.y = tile rows, int pixel offsets
    return 0;
}

dim3 edge_grid(int C, int H, int W) { return dim3((W + TW - 1) / TW, (H + TH - 1) / TH, C); }

// ---- tv_loss --------------------------------------------------------------------------------------------------
constexpr int TV_PER = NT * 8;          // elements of one plane per CTA

struct TvScale {
    double n_h, n_w;                    // B (H-1) W vertical and B H (W-1) horizontal differences (the two means)
};
TvScale tv_scale(int B, int H, int W) { return {(double)B * (H - 1) * W, (double)B * H * (W - 1)}; }

// grid (ceil(H W / TV_PER), B); partial = (sum of squared vertical differences) / n_h + (horizontal) / n_w
__global__ void __launch_bounds__(NT) tv_fwd_kernel(int H, int W, const float* __restrict__ x, double inv_h,
                                                    double inv_w, double* __restrict__ partial) {
    const unsigned HW = (unsigned)H * (unsigned)W;
    const float* p = x + (size_t)blockIdx.y * HW;
    double ah = 0.0, aw = 0.0;
    for (unsigned i = blockIdx.x * TV_PER + threadIdx.x, e = min(HW, (blockIdx.x + 1) * TV_PER); i < e; i += NT) {
        const unsigned r = i / (unsigned)W, c = i - r * (unsigned)W;
        const float v = __ldg(p + i);
        if (r + 1 < (unsigned)H) { const float d = sub_(__ldg(p + i + W), v); ah += (double)mul_(d, d); }
        if (c + 1 < (unsigned)W) { const float d = sub_(__ldg(p + i + 1), v); aw += (double)mul_(d, d); }
    }
    cta_partial<NT>(ah * inv_h + aw * inv_w, partial + (size_t)blockIdx.y * gridDim.x + blockIdx.x);
}

// dL/dx[i] = 2 g / n_h (d_up - d_down) + 2 g / n_w (d_left - d_right), each difference present where it exists
__global__ void __launch_bounds__(NT) tv_bwd_kernel(int H, int W, const float* __restrict__ x, const float* __restrict__ g,
                                                    float n_h, float n_w, float* __restrict__ dx) {
    const unsigned HW = (unsigned)H * (unsigned)W;
    const size_t plane = (size_t)blockIdx.y * HW;
    const float* p = x + plane;
    const float th = mul_(2.0f, div_(g[0], n_h)), tw = mul_(2.0f, div_(g[0], n_w));
    for (unsigned i = blockIdx.x * TV_PER + threadIdx.x, e = min(HW, (blockIdx.x + 1) * TV_PER); i < e; i += NT) {
        const unsigned r = i / (unsigned)W, c = i - r * (unsigned)W;
        const float v = __ldg(p + i);
        float a = 0.f, b = 0.f;
        if (r > 0) a = sub_(v, __ldg(p + i - W));
        if (r + 1 < (unsigned)H) a = sub_(a, sub_(__ldg(p + i + W), v));
        if (c > 0) b = sub_(v, __ldg(p + i - 1));
        if (c + 1 < (unsigned)W) b = sub_(b, sub_(__ldg(p + i + 1), v));
        dx[plane + i] = add_(mul_(th, a), mul_(tw, b));
    }
}

int check_tv(int B, int H, int W) {
    if (B <= 0 || H < 2 || W < 2) return R3DG_ERR_BAD_ARG;      // H or W of 1: the reference's mean of nothing
    if (B > 65535 || (long long)H * W > (1LL << 31) - 1) return R3DG_ERR_UNSUPPORTED;   // grid.y = planes
    return 0;
}

dim3 tv_grid(int B, int H, int W) { return dim3((unsigned)(((long long)H * W + TV_PER - 1) / TV_PER), B); }

size_t partial_bytes(dim3 gr) { return ((size_t)gr.x * gr.y * gr.z * sizeof(double) + 255) & ~(size_t)255; }

}  // namespace

size_t edge_aware_tmp_bytes(int Cd, int Ci, int H, int W) {
    if (check_edge(Cd, Ci, H, W) != 0) return 0;
    return partial_bytes(edge_grid(max(Cd, Ci), H, W));
}

int launch_edge_aware_forward(int Cd, int Ci, int H, int W, const float* data, const float* img, float* out, void* tmp,
                              size_t tmp_bytes, cudaStream_t stream) {
    const int rc = check_edge(Cd, Ci, H, W);
    if (rc != 0) return rc;
    if (!data || !img || !out || !tmp || tmp_bytes < edge_aware_tmp_bytes(Cd, Ci, H, W)) return R3DG_ERR_BAD_ARG;
    const int C = max(Cd, Ci);
    const dim3 gr = edge_grid(C, H, W);
    edge_fwd_kernel<<<gr, NT, 0, stream>>>(Cd, Ci, H, W, data, img, (double*)tmp);
    R3DG_CUDA_TRY(cudaGetLastError());
    reduce_partials_kernel<<<1, kReduceNT, 0, stream>>>((const double*)tmp, (long long)gr.x * gr.y * gr.z,
                                                        (double)C * H * W, out);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_edge_aware_backward(int Cd, int Ci, int H, int W, const float* data, const float* img, const float* dL_dout,
                               float* dL_ddata, float* dL_dimg, cudaStream_t stream) {
    const int rc = check_edge(Cd, Ci, H, W);
    if (rc != 0) return rc;
    if (!data || !img || !dL_dout || (!dL_ddata && !dL_dimg)) return R3DG_ERR_BAD_ARG;
    const int C = max(Cd, Ci);
    const dim3 gr = edge_grid(Cd == Ci ? C : 1, H, W);
    edge_bwd_kernel<<<gr, NT, 0, stream>>>(C, Cd, Ci, H, W, data, img, dL_dout, (float)((double)C * H * W), dL_ddata,
                                           dL_dimg);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

size_t tv_tmp_bytes(int B, int H, int W) {
    if (check_tv(B, H, W) != 0) return 0;
    return partial_bytes(tv_grid(B, H, W));
}

int launch_tv_forward(int B, int H, int W, const float* x, float* out, void* tmp, size_t tmp_bytes, cudaStream_t stream) {
    const int rc = check_tv(B, H, W);
    if (rc != 0) return rc;
    if (!x || !out || !tmp || tmp_bytes < tv_tmp_bytes(B, H, W)) return R3DG_ERR_BAD_ARG;
    const dim3 gr = tv_grid(B, H, W);
    const TvScale n = tv_scale(B, H, W);
    tv_fwd_kernel<<<gr, NT, 0, stream>>>(H, W, x, 1.0 / n.n_h, 1.0 / n.n_w, (double*)tmp);
    R3DG_CUDA_TRY(cudaGetLastError());
    reduce_partials_kernel<<<1, kReduceNT, 0, stream>>>((const double*)tmp, (long long)gr.x * gr.y, 1.0, out);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_tv_backward(int B, int H, int W, const float* x, const float* dL_dout, float* dL_dx, cudaStream_t stream) {
    const int rc = check_tv(B, H, W);
    if (rc != 0) return rc;
    if (!x || !dL_dout || !dL_dx) return R3DG_ERR_BAD_ARG;
    const TvScale n = tv_scale(B, H, W);
    tv_bwd_kernel<<<tv_grid(B, H, W), NT, 0, stream>>>(H, W, x, dL_dout, (float)n.n_h, (float)n.n_w, dL_dx);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
