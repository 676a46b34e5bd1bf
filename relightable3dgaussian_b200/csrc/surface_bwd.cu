// Adjoint of surface_normal_kernel (composite.cu): the cotangents of the pseudo-normal and surface-xyz images become
// extra cotangents of the depth and opacity images, which the backward compositor then consumes unchanged, plus the
// pseudo-normal's term of dL/dviewmatrix.  DESIGN.md §4.9.
//
// In the forward's names, per pixel: d = depth / max(o, 1e-7), P = (a d, b d, d) with a = (x - cx) / fx,
// b = (y - cy) / fy; ga, gb the two Sobel stencils over the clamped 3x3 window of P; n = ga x gb, N = -n / |n|;
// normal_k = sum_i V[4k + i] N_i (zero where !(|n| > 0)); surface_xyz = P.
// The scatter of a pixel's stencil gradients onto its neighbours is written as a gather: every pixel q sums, in a fixed
// order, the contributions of the stencil slots of its 3x3 neighbours that land on q after the border clamp.  No
// atomics: the result is bitwise reproducible.
#include "common.cuh"
#include "kernels.h"

namespace r3dg {
namespace {

constexpr int kTW = 32, kTH = 8;                       // pixel tile of one CTA, one thread per pixel
constexpr int kPW = kTW + 4, kPH = kTH + 4;            // surface points: the tile plus a 2-pixel halo
constexpr int kRW = kTW + 2, kRH = kTH + 2;            // stencil gradients: the tile plus a 1-pixel ring

struct SurfaceBwdParams {
    int W, H, nblk;
    float focal_x, focal_y, cx, cy;
    const float* V;                                    // the view's viewmatrix [16]
    const float *opacity, *depth;                      // the forward's images [H,W]
    const float *g_normal, *g_xyz;                     // [3,H,W] or null (zero)
    const float *g_depth, *g_opacity;                  // the caller's cotangents [H,W]
    float *out_depth, *out_opacity;                    // the combined cotangents [H,W]
    float* cam_part;                                   // [9][nblk] per-CTA sums of g_o_k N_i, or null
};

// stencil weights of slot (dy, dx) in the forward's ga (horizontal) and gb (vertical) Sobel sums
__device__ __forceinline__ float w_a(int dy, int dx) { return (float)dx * (dy == 0 ? 0.25f : 0.125f); }
__device__ __forceinline__ float w_b(int dy, int dx) { return (float)dy * (dx == 0 ? 0.25f : 0.125f); }

__global__ void __launch_bounds__(256) surface_bwd_kernel(SurfaceBwdParams p) {
    __shared__ double sP[3][kPH][kPW];
    __shared__ double sDa[3][kRH][kRW], sDb[3][kRH][kRW];
    __shared__ float sCam[8][9];
    const int t = threadIdx.x, x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
    const int W = p.W, H = p.H;
    const size_t HW = (size_t)H * W;

    // 1. surface points of the tile and a 2-pixel halo (positions outside the image are never read).  The stencil
    // takes differences of neighbouring points that are ~1/W of the points themselves, so steps 1 to 3 run in fp64
    // from the forward's fp32 images: in fp32 those differences would lose about log2(W) bits.  The stencil gradients
    // stay in fp64 shared memory too, because the gather of step 3 is again a difference of neighbours.
    for (int r = t; r < kPW * kPH; r += 256) {
        const int ly = r / kPW, lx = r % kPW, gx = x0 - 2 + lx, gy = y0 - 2 + ly;
        double P0 = 0.0, P1 = 0.0, P2 = 0.0;
        if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
            const size_t q = (size_t)W * gy + gx;
            const double d = (double)p.depth[q] / (double)fmaxf(p.opacity[q], 0.0000001f);
            P0 = ((double)gx - p.cx) / p.focal_x * d;
            P1 = ((double)gy - p.cy) / p.focal_y * d;
            P2 = d;
        }
        sP[0][ly][lx] = P0; sP[1][ly][lx] = P1; sP[2][ly][lx] = P2;
    }
    __syncthreads();

    // 2. per pixel of the tile and a 1-pixel ring: dL/dga and dL/dgb; the tile's pixels also add g_o_k N_i to this
    // thread's camera sums (items in a fixed order per thread)
    float cam[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) cam[k] = 0.0f;
    for (int r = t; r < kRW * kRH; r += 256) {
        const int ry = r / kRW, rx = r % kRW, x = x0 - 1 + rx, y = y0 - 1 + ry;
        double da[3] = {0.0, 0.0, 0.0}, db[3] = {0.0, 0.0, 0.0};
        if (p.g_normal && x >= 0 && x < W && y >= 0 && y < H) {
            const int xm = x == 0 ? 0 : x - 1, xp = x == W - 1 ? W - 1 : x + 1;
            const int ym = y == 0 ? 0 : y - 1, yp = y == H - 1 ? H - 1 : y + 1;
            const int cxm = xm - x0 + 2, cx0 = x - x0 + 2, cxp = xp - x0 + 2;
            const int cym = ym - y0 + 2, cy0 = y - y0 + 2, cyp = yp - y0 + 2;
            double ga[3], gb[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                ga[i] = 0.125 * (sP[i][cym][cxp] - sP[i][cym][cxm] + sP[i][cyp][cxp] - sP[i][cyp][cxm]) +
                        0.25 * (sP[i][cy0][cxp] - sP[i][cy0][cxm]);
                gb[i] = 0.125 * (sP[i][cyp][cxm] - sP[i][cym][cxm] + sP[i][cyp][cxp] - sP[i][cym][cxp]) +
                        0.25 * (sP[i][cyp][cx0] - sP[i][cym][cx0]);
            }
            const double n0 = ga[1] * gb[2] - ga[2] * gb[1];
            const double n1 = ga[2] * gb[0] - ga[0] * gb[2];
            const double n2 = ga[0] * gb[1] - ga[1] * gb[0];
            const double norm = sqrt(n0 * n0 + n1 * n1 + n2 * n2);
            if (norm > 0.0) {
                const size_t q = (size_t)W * y + x;
                const float go[3] = {p.g_normal[q], p.g_normal[HW + q], p.g_normal[2 * HW + q]};
                const float* V = p.V;
                double gN[3];                                                       // g_N = M^T g_o
#pragma unroll
                for (int i = 0; i < 3; ++i) gN[i] = (double)V[i] * go[0] + (double)V[4 + i] * go[1] + (double)V[8 + i] * go[2];
                const double inv = 1.0 / norm;
                const double h0 = n0 * inv, h1 = n1 * inv, h2 = n2 * inv;
                const double hg = h0 * gN[0] + h1 * gN[1] + h2 * gN[2];
                // dL/dn = -(g_N - n^ (n^ . g_N)) / |n|
                const double dn0 = (h0 * hg - gN[0]) * inv, dn1 = (h1 * hg - gN[1]) * inv, dn2 = (h2 * hg - gN[2]) * inv;
                da[0] = gb[1] * dn2 - gb[2] * dn1;                         // dga = gb x dL/dn
                da[1] = gb[2] * dn0 - gb[0] * dn2;
                da[2] = gb[0] * dn1 - gb[1] * dn0;
                db[0] = dn1 * ga[2] - dn2 * ga[1];                         // dgb = dL/dn x ga
                db[1] = dn2 * ga[0] - dn0 * ga[2];
                db[2] = dn0 * ga[1] - dn1 * ga[0];
                if (rx >= 1 && rx <= kTW && ry >= 1 && ry <= kTH) {                // a pixel of the tile: camera term
                    const float N[3] = {(float)(-h0), (float)(-h1), (float)(-h2)};
#pragma unroll
                    for (int k = 0; k < 3; ++k)
#pragma unroll
                        for (int i = 0; i < 3; ++i) cam[3 * k + i] = fma_(go[k], N[i], cam[3 * k + i]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) { sDa[i][ry][rx] = da[i]; sDb[i][ry][rx] = db[i]; }
    }
    __syncthreads();

    // 3. / 4. gather dL/dP at pixel q, then the combined depth and opacity cotangents
    const int qx = x0 + (t & 31), qy = y0 + (t >> 5);
    if (qx < W && qy < H) {
        const size_t q = (size_t)W * qy + qx;
        double gP[3];                                   // fp64 as well: the gather is again a difference of neighbours
#pragma unroll
        for (int i = 0; i < 3; ++i) gP[i] = p.g_xyz ? (double)p.g_xyz[i * HW + q] : 0.0;
        if (p.g_normal) {
            for (int ty = -1; ty <= 1; ++ty) {
                const int py = qy + ty;
                if (py < 0 || py >= H) continue;
                for (int tx = -1; tx <= 1; ++tx) {
                    const int px = qx + tx;
                    if (px < 0 || px >= W) continue;
                    const int ry = py - y0 + 1, rx = px - x0 + 1;
                    float ca = 0.0f, cb = 0.0f;         // summed weights of p's slots that land on q after the clamp
                    for (int sy = -1; sy <= 1; ++sy) {
                        if (min(max(py + sy, 0), H - 1) != qy) continue;
                        for (int sx = -1; sx <= 1; ++sx) {
                            if (min(max(px + sx, 0), W - 1) != qx) continue;
                            ca += w_a(sy, sx);          // multiples of 1/8: exact
                            cb += w_b(sy, sx);
                        }
                    }
#pragma unroll
                    for (int i = 0; i < 3; ++i) gP[i] += ca * sDa[i][ry][rx] + cb * sDb[i][ry][rx];
                }
            }
        }
        const float o = p.opacity[q], depth = p.depth[q];
        const double a = ((double)qx - p.cx) / p.focal_x, b = ((double)qy - p.cy) / p.focal_y;
        const double dd = a * gP[0] + b * gP[1] + gP[2];                            // dL/dd
        const double om = fmaxf(o, 0.0000001f);
        p.out_depth[q] = (float)(p.g_depth[q] + dd / om);
        p.out_opacity[q] = o > 0.0000001f ? (float)(p.g_opacity[q] - dd * depth / ((double)o * o)) : p.g_opacity[q];
    }

    // camera term: the CTA's 9 sums in a fixed order (a shuffle tree per warp, then the warps in order)
    if (p.cam_part) {
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            float s = cam[k];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) s = add_(s, __shfl_down_sync(0xffffffffu, s, off));
            if ((t & 31) == 0) sCam[t >> 5][k] = s;
        }
        __syncthreads();
        if (t < 9) {
            float s = sCam[0][t];
            for (int w = 1; w < 8; ++w) s = add_(s, sCam[w][t]);
            p.cam_part[(size_t)t * p.nblk + blockIdx.y * gridDim.x + blockIdx.x] = s;
        }
    }
}

// dL/dviewmatrix[v][4k + i] += the sum of view v's CTA partials of entry 3k + i, in CTA order: one warp per entry
__global__ void __launch_bounds__(32) surface_cam_sum_kernel(const float* __restrict__ part, int nblk,
                                                             float* __restrict__ dL_dviewmatrix) {
    const int v = blockIdx.y, e = blockIdx.x, lane = threadIdx.x;
    const float* col = part + ((size_t)v * 9 + e) * nblk;
    float s = 0.0f;
    for (int j = lane; j < nblk; j += 32) s = add_(s, col[j]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s = add_(s, __shfl_down_sync(0xffffffffu, s, off));
    if (lane == 0) {
        float* o = dL_dviewmatrix + (size_t)v * 16 + 4 * (e / 3) + e % 3;
        *o = add_(*o, s);
    }
}

}  // namespace

int surface_grad_blocks(int W, int H) { return ((W < 1 ? 1 : W) + kTW - 1) / kTW * (((H < 1 ? 1 : H) + kTH - 1) / kTH); }

int launch_surface_backward(const r3dg_raster_bwd_args& a, int V, float* planes, float* cam_part, cudaStream_t stream) {
    const size_t HW = (size_t)a.H * a.W;
    const int nblk = surface_grad_blocks(a.W, a.H);
    const dim3 grid((a.W + kTW - 1) / kTW, (a.H + kTH - 1) / kTH);
    for (int v = 0; v < V; ++v) {                      // each view with its own intrinsics and viewmatrix
        float tan_fovx = a.tan_fovx, tan_fovy = a.tan_fovy, cx = a.cx, cy = a.cy;
        view_cam(V, a.view_cams, v, tan_fovx, tan_fovy, cx, cy);
        SurfaceBwdParams p;
        p.W = a.W; p.H = a.H; p.nblk = nblk;
        p.focal_y = a.H / (2.0f * tan_fovy); p.focal_x = a.W / (2.0f * tan_fovx);   // as the forward computes them
        p.cx = cx; p.cy = cy;
        p.V = a.viewmatrix + 16 * v;
        p.opacity = a.fwd_opacity + v * HW; p.depth = a.fwd_depth + v * HW;
        p.g_normal = a.dL_dout_normal ? a.dL_dout_normal + 3 * v * HW : nullptr;
        p.g_xyz = a.dL_dout_surface_xyz ? a.dL_dout_surface_xyz + 3 * v * HW : nullptr;
        p.g_depth = a.dL_dout_depth + v * HW; p.g_opacity = a.dL_dout_opacity + v * HW;
        p.out_depth = planes + v * HW; p.out_opacity = planes + (V + v) * HW;
        p.cam_part = cam_part ? cam_part + (size_t)v * 9 * nblk : nullptr;
        surface_bwd_kernel<<<grid, 256, 0, stream>>>(p);
    }
    return -(int)cudaGetLastError();
}

int launch_surface_cam_sum(const float* cam_part, int nblk, int V, float* dL_dviewmatrix, cudaStream_t stream) {
    surface_cam_sum_kernel<<<dim3(9, V), 32, 0, stream>>>(cam_part, nblk, dL_dviewmatrix);
    return -(int)cudaGetLastError();
}

}  // namespace r3dg
