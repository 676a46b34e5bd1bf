// Bilateral-grid colour correction (Wang et al., "Bilateral Guided Radiance Field Processing", SIGGRAPH 2024; gsplat's
// BilateralGrid / slice): every pixel of image n gets the 3x4 affine colour transform A trilinearly interpolated from
// grids[ids[n]] ([12, L, GY, GX]) at (x, y, luma), out_c = A[4c..4c+2] . rgb + A[4c+3].
//
// Coordinates (align_corners, border padding): ix = (px + 0.5) (GX - 1) / W, iy likewise, iz = luma (L - 1) clamped to
// [0, L - 1].  The cell of a coordinate is i0 = min(floor(i), size - 2), t = i - i0 in [0, 1], so both corners of a
// cell are distinct nodes.  Interpolation is nested lerps v0 + t (v1 - v0), x, then y, then z: a constant grid gives
// its value exactly, and the identity grid returns rgb bit for bit.
//
// Pixels are cut into TS x TS tiles.  The nodes one tile touches (a few xy nodes x L x 12 coefficients) are staged in
// shared memory with the coefficients innermost, so a corner is three 16-byte loads.
//   forward : one CTA of 256 threads per tile, one pass over the pixels (12 B read, 12 B written per pixel);
//   backward: one warp per tile.  Each lane owns one pixel column: it reads rgb and dL/dout, writes dL/drgb, and hands
//             its pixel to the warp's grid accumulation, where lane q owns the (xy corner, z node) row q of the current
//             xy cell in 12 registers and the pixels are added in a fixed order.  A change of cell adds the rows to the
//             tile's partial sub-grid in shared memory, which ends as a slab of the workspace;
//   reduce  : one thread per grid coefficient sums, in a fixed order (views, tile rows, tile columns), the slabs of the
//             tiles that touch it.
// No float atomics anywhere, so every result is bitwise reproducible run to run.
#include "common.cuh"
#include "kernels.h"

namespace r3dg {
namespace {

constexpr int TS = 32;                 // tile edge in pixels
constexpr int FWD_NT = 256;
constexpr int MAX_NODES = 1024;        // staged nodes per tile (48 KB of coefficients)
constexpr int MAX_L = 16;              // 4 L (xy corner, z node) rows over the 32 lanes of the backward warp: R <= 2

// Grid coordinate of pixel p on an axis of npix pixels and n nodes: fl(fl((p + 0.5) (n - 1)) / npix), each step
// correctly rounded.  The product is not always exact (e.g. npix = 100003, n = 1024), so the result can lie about an
// fp32 ulp from the exact coordinate; every step is monotone, so it stays in [0, n - 1] and monotone in p, and all
// tiles agree on each pixel's cell.
__device__ __forceinline__ float pix_coord(int p, int n, int npix) {
    return div_(mul_((float)p + 0.5f, (float)(n - 1)), (float)npix);
}
__device__ __forceinline__ int cell_of(float c, int n) { return min((int)c, n - 2); }   // c >= 0

// First node and node count of the tile starting at pixel t0 on an axis
__device__ __forceinline__ void tile_nodes(int t0, int n, int npix, int& c0, int& cnt) {
    const int t1 = min(t0 + TS, npix) - 1;
    c0 = cell_of(pix_coord(t0, n, npix), n);
    cnt = cell_of(pix_coord(t1, n, npix), n) + 2 - c0;
}

// Host bound on tile_nodes' count: the coordinate advances by (TS - 1)(n - 1) / npix across a tile, so the cells differ
// by at most floor of that + 1; +1 more absorbs the rounding of the two ends.
int max_tile_nodes(int n, int npix) {
    return min(n, (int)((double)(TS - 1) * (n - 1) / npix + 1e-3) + 3);
}

struct Shape {
    int N, H, W, GX, GY, L;
    int nx, ny;                       // host bounds of the staged sub-grid
    size_t nodes() const { return (size_t)nx * ny * L; }
    int tiles_x() const { return (W + TS - 1) / TS; }
    int tiles_y() const { return (H + TS - 1) / TS; }
};

int check(int G, int N, int H, int W, int GX, int GY, int L, Shape& s) {
    if (G <= 0 || N <= 0 || H <= 0 || W <= 0 || GX < 2 || GY < 2 || L < 2) return R3DG_ERR_BAD_ARG;
    if (N > 65535 || (long long)H * W > (1LL << 31) - 1 || (H + TS - 1) / TS > 65535 || W > (1 << 20) || H > (1 << 20) ||
        GX > 1024 || GY > 1024 || L > MAX_L || (long long)G * 12 * L * GY * GX > (1LL << 31) - 1)
        return R3DG_ERR_UNSUPPORTED;
    s = {N, H, W, GX, GY, L, max_tile_nodes(GX, W), max_tile_nodes(GY, H)};
    if (s.nodes() > (size_t)MAX_NODES) return R3DG_ERR_UNSUPPORTED;
    return 0;
}

// Stage the tile's sub-grid of grid g: s[((n ny + y) nx + x) 12 + k] = grid[k][n][cy0 + y][cx0 + x]
__device__ __forceinline__ void stage_subgrid(float* s, const float* __restrict__ grid, int GX, int GY, int L, int cx0,
                                              int nx, int cy0, int ny, int nth) {
    const int total = nx * ny * L * 12;
    for (int i = threadIdx.x; i < total; i += nth) {
        int r = i;
        const int x = r % nx; r /= nx;
        const int y = r % ny; r /= ny;
        const int n = r % L;
        const int k = r / L;
        s[((n * ny + y) * nx + x) * 12 + k] = __ldg(grid + ((size_t)(k * L + n) * GY + cy0 + y) * GX + cx0 + x);
    }
}

__device__ __forceinline__ float lerp_(float a, float b, float t) { return fma_(t, sub_(b, a), a); }

// The 12 coefficients of z slice n, bilinear in (x, y) over the cell whose low corner is sub-grid node (xr, yr)
__device__ __forceinline__ void slice_xy(const float* s, int nx, int ny, int n, int xr, int yr, float tx, float ty,
                                         float (&S)[12]) {
    const float4* p00 = reinterpret_cast<const float4*>(s + ((n * ny + yr) * nx + xr) * 12);
    const float4* p01 = p00 + 3;                      // x + 1
    const float4* p10 = p00 + 3 * nx;                 // y + 1
    const float4* p11 = p10 + 3;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        const float4 a = p00[q], b = p01[q], c = p10[q], d = p11[q];
        S[4 * q + 0] = lerp_(lerp_(a.x, b.x, tx), lerp_(c.x, d.x, tx), ty);
        S[4 * q + 1] = lerp_(lerp_(a.y, b.y, tx), lerp_(c.y, d.y, tx), ty);
        S[4 * q + 2] = lerp_(lerp_(a.z, b.z, tx), lerp_(c.z, d.z, tx), ty);
        S[4 * q + 3] = lerp_(lerp_(a.w, b.w, tx), lerp_(c.w, d.w, tx), ty);
    }
}

__device__ __forceinline__ float luma(float r, float g, float b) {
    return fma_(0.114f, b, fma_(0.587f, g, mul_(0.299f, r)));
}

// z coordinate of a luma value: the clamped coordinate's cell and weight, and whether the unclamped one lies strictly
// inside (torch's clip_coordinates_set_grad: the luma gradient is 0 at and beyond the border)
__device__ __forceinline__ void z_coord(float z, int L, int& z0, float& tz, bool& inside) {
    const float iz = mul_(z, (float)(L - 1));
    inside = iz > 0.0f && iz < (float)(L - 1);
    const float c = fminf(fmaxf(iz, 0.0f), (float)(L - 1));      // NaN -> 0
    z0 = cell_of(c, L);
    tz = sub_(c, (float)z0);
}

__device__ __forceinline__ float affine_row(const float (&A)[12], int c, float r, float g, float b) {
    return fma_(A[4 * c], r, fma_(A[4 * c + 1], g, fma_(A[4 * c + 2], b, A[4 * c + 3])));
}

__global__ void __launch_bounds__(FWD_NT) bilagrid_fwd_kernel(int H, int W, int GX, int GY, int L,
                                                              const float* __restrict__ grids,
                                                              const int* __restrict__ ids, const float* __restrict__ rgb,
                                                              float* __restrict__ out) {
    extern __shared__ float4 smem4[];
    float* s = reinterpret_cast<float*>(smem4);
    const int v = blockIdx.z, x0 = blockIdx.x * TS, y0 = blockIdx.y * TS;
    int cx0, nx, cy0, ny;
    tile_nodes(x0, GX, W, cx0, nx);
    tile_nodes(y0, GY, H, cy0, ny);
    const float* grid = grids + (size_t)__ldg(ids + v) * 12 * L * GY * GX;
    stage_subgrid(s, grid, GX, GY, L, cx0, nx, cy0, ny, FWD_NT);
    __syncthreads();
    const size_t HW = (size_t)H * W;
    const float* in = rgb + (size_t)v * 3 * HW;
    float* o = out + (size_t)v * 3 * HW;
    const int px = x0 + (threadIdx.x & (TS - 1));
    if (px >= W) return;
    const float ix = pix_coord(px, GX, W);
    const int xc = cell_of(ix, GX);
    const float tx = sub_(ix, (float)xc);
    for (int py = y0 + (threadIdx.x >> 5); py < min(y0 + TS, H); py += FWD_NT / TS) {
        const float iy = pix_coord(py, GY, H);
        const int yc = cell_of(iy, GY);
        const float ty = sub_(iy, (float)yc);
        const size_t i = (size_t)py * W + px;
        const float r = __ldg(in + i), g = __ldg(in + HW + i), b = __ldg(in + 2 * HW + i);
        int z0; float tz; bool inside;
        z_coord(luma(r, g, b), L, z0, tz, inside);
        float S0[12], S1[12], A[12];
        slice_xy(s, nx, ny, z0, xc - cx0, yc - cy0, tx, ty, S0);
        slice_xy(s, nx, ny, z0 + 1, xc - cx0, yc - cy0, tx, ty, S1);
#pragma unroll
        for (int k = 0; k < 12; ++k) A[k] = lerp_(S0[k], S1[k], tz);
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c * HW + i] = affine_row(A, c, r, g, b);
    }
}

// Per-pixel record handed from the lane that owns the pixel to the warp's grid accumulation
struct alignas(16) PixRec {
    int xr; float tx; int z0; float tz;          // x cell (sub-grid relative), weight; z cell, weight
    float d0, d1, d2, r;                         // dL/dout, rgb
    float g, b, pad0, pad1;
};

// R = (xy corner, z node) rows per lane (4 L <= 32 R); GRID: accumulate dL/dgrids partials
template <int R, bool GRID>
__global__ void __launch_bounds__(32) bilagrid_bwd_kernel(int H, int W, int GX, int GY, int L, int slab,
                                                          const float* __restrict__ grids, const int* __restrict__ ids,
                                                          const float* __restrict__ rgb, const float* __restrict__ dout,
                                                          float* __restrict__ drgb, float* __restrict__ partials) {
    extern __shared__ float4 smem4[];
    const int lane = threadIdx.x;
    const int v = blockIdx.z, x0 = blockIdx.x * TS, y0 = blockIdx.y * TS;
    int cx0, nx, cy0, ny;
    tile_nodes(x0, GX, W, cx0, nx);
    tile_nodes(y0, GY, H, cy0, ny);
    const int nodes12 = nx * ny * L * 12;
    float* s = reinterpret_cast<float*>(smem4);
    float* part = s + nodes12;                                   // 16-byte aligned: nodes12 is a multiple of 4
    PixRec* rec = reinterpret_cast<PixRec*>(part + (GRID ? nodes12 : 0));
    const float* grid = grids + (size_t)__ldg(ids + v) * 12 * L * GY * GX;
    stage_subgrid(s, grid, GX, GY, L, cx0, nx, cy0, ny, 32);
    if (GRID)
        for (int i = lane; i < nodes12; i += 32) part[i] = 0.0f;
    __syncwarp();

    const size_t HW = (size_t)H * W;
    const float* in = rgb + (size_t)v * 3 * HW;
    const float* go = dout + (size_t)v * 3 * HW;
    float* dr = drgb ? drgb + (size_t)v * 3 * HW : nullptr;
    const int px = x0 + lane;
    const bool live = px < W;
    const float ix = pix_coord(min(px, W - 1), GX, W);
    const int xc = cell_of(ix, GX);
    const float tx = sub_(ix, (float)xc);
    const float lscale = (float)(L - 1);

    // lane row q = lane + 32 j: z node q % L of xy corner q / L (bit 0: x + 1, bit 1: y + 1); rows >= 4 L are idle
    int rn[R], rbx[R], rby[R];
    bool ron[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
        const int q = lane + 32 * j;
        ron[j] = q < 4 * L;
        rn[j] = q % L; rbx[j] = (q / L) & 1; rby[j] = (q / L) >> 1;
    }
    float acc[R][12];
#pragma unroll
    for (int j = 0; j < R; ++j)
#pragma unroll
        for (int k = 0; k < 12; ++k) acc[j][k] = 0.0f;
    int cur_x = -1, cur_y = -1;                      // xy cell of the rows being accumulated (sub-grid relative)
    auto flush = [&]() {
        // consecutive flushes of one pixel row share part entries across lanes (corner bx = 1 of cell X is corner
        // bx = 0 of cell X + 1), so the previous flush's stores must be visible first
        __syncwarp();
        if (cur_x < 0) return;
#pragma unroll
        for (int j = 0; j < R; ++j) {
            if (ron[j]) {
                float4* p = reinterpret_cast<float4*>(part + ((rn[j] * ny + cur_y + rby[j]) * nx + cur_x + rbx[j]) * 12);
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    float4 a = p[q];
                    a.x = add_(a.x, acc[j][4 * q]); a.y = add_(a.y, acc[j][4 * q + 1]);
                    a.z = add_(a.z, acc[j][4 * q + 2]); a.w = add_(a.w, acc[j][4 * q + 3]);
                    p[q] = a;
                }
            }
#pragma unroll
            for (int k = 0; k < 12; ++k) acc[j][k] = 0.0f;
        }
    };

    for (int py = y0; py < min(y0 + TS, H); ++py) {
        const float iy = pix_coord(py, GY, H);
        const int yc = cell_of(iy, GY);
        const float ty = sub_(iy, (float)yc);
        const size_t i = (size_t)py * W + px;
        float r = 0.f, g = 0.f, b = 0.f, d0 = 0.f, d1 = 0.f, d2 = 0.f;
        if (live) {
            r = __ldg(in + i); g = __ldg(in + HW + i); b = __ldg(in + 2 * HW + i);
            d0 = __ldg(go + i); d1 = __ldg(go + HW + i); d2 = __ldg(go + 2 * HW + i);
        }
        int z0; float tz; bool inside;
        z_coord(luma(r, g, b), L, z0, tz, inside);
        if (dr && live) {
            float S0[12], S1[12];
            slice_xy(s, nx, ny, z0, xc - cx0, yc - cy0, tx, ty, S0);
            slice_xy(s, nx, ny, z0 + 1, xc - cx0, yc - cy0, tx, ty, S1);
            float gz = 0.0f;                          // dL/diz = sum_c dout_c (dA_c/diz . (rgb, 1)), dA/diz = S1 - S0
            float gr = 0.0f, gg = 0.0f, gb = 0.0f;    // A^T dL/dout
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float d = c == 0 ? d0 : (c == 1 ? d1 : d2);
                float D[4], A[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    D[j] = sub_(S1[4 * c + j], S0[4 * c + j]);
                    A[j] = lerp_(S0[4 * c + j], S1[4 * c + j], tz);
                }
                gz = fma_(d, fma_(D[0], r, fma_(D[1], g, fma_(D[2], b, D[3]))), gz);
                gr = fma_(A[0], d, gr); gg = fma_(A[1], d, gg); gb = fma_(A[2], d, gb);
            }
            if (inside) {
                const float gl = mul_(gz, lscale);
                gr = fma_(0.299f, gl, gr); gg = fma_(0.587f, gl, gg); gb = fma_(0.114f, gl, gb);
            }
            dr[i] = gr; dr[HW + i] = gg; dr[2 * HW + i] = gb;
        }
        if (GRID) {
            rec[lane] = PixRec{xc - cx0, tx, z0, tz, d0, d1, d2, r, g, b, 0.f, 0.f};
            __syncwarp();
            const int yr = yc - cy0;
            float wy[R];
#pragma unroll
            for (int j = 0; j < R; ++j) wy[j] = rby[j] ? ty : sub_(1.0f, ty);
            const int np = min(TS, W - x0);
            for (int p = 0; p < np; ++p) {
                const float4* rp = reinterpret_cast<const float4*>(rec + p);
                const float4 h = rp[0], c1 = rp[1], c2 = rp[2];
                const int pxr = __float_as_int(h.x), pz0 = __float_as_int(h.z);
                if (pxr != cur_x || yr != cur_y) { flush(); cur_x = pxr; cur_y = yr; }
#pragma unroll
                for (int j = 0; j < R; ++j) {
                    const float wx = rbx[j] ? h.y : sub_(1.0f, h.y);
                    const float wz = rn[j] == pz0 ? sub_(1.0f, h.w) : (rn[j] == pz0 + 1 ? h.w : 0.0f);
                    const float w = mul_(mul_(wx, wy[j]), wz);
                    const float a0 = mul_(w, c1.x), a1 = mul_(w, c1.y), a2 = mul_(w, c1.z);
                    const float in3[3] = {c1.w, c2.x, c2.y};
#pragma unroll
                    for (int q = 0; q < 3; ++q) {
                        acc[j][q] = fma_(a0, in3[q], acc[j][q]);
                        acc[j][4 + q] = fma_(a1, in3[q], acc[j][4 + q]);
                        acc[j][8 + q] = fma_(a2, in3[q], acc[j][8 + q]);
                    }
                    acc[j][3] = add_(acc[j][3], a0); acc[j][7] = add_(acc[j][7], a1); acc[j][11] = add_(acc[j][11], a2);
                }
            }
            __syncwarp();
        }
    }
    if (GRID) {
        flush();
        __syncwarp();
        float* dst = partials + (((size_t)v * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * slab;
        for (int i = lane; i < nodes12; i += 32) dst[i] = part[i];
    }
}

// dL/dgrids[g][k][n][y][x] = sum over the views with id g, the tile rows, then the tile columns whose sub-grid holds
// (x, y), of that slab's entry.  Unused grids get 0.
__global__ void bilagrid_reduce_kernel(int G, int N, int H, int W, int GX, int GY, int L, int slab,
                                       const int* __restrict__ ids, const float* __restrict__ partials,
                                       float* __restrict__ dgrids) {
    const long long total = (long long)G * 12 * L * GY * GX;
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    long long r = e;
    const int x = (int)(r % GX); r /= GX;
    const int y = (int)(r % GY); r /= GY;
    const int n = (int)(r % L); r /= L;
    const int k = (int)(r % 12);
    const int g = (int)(r / 12);
    const int tiles_x = (W + TS - 1) / TS, tiles_y = (H + TS - 1) / TS;
    float sum = 0.0f;
    for (int v = 0; v < N; ++v) {
        if (__ldg(ids + v) != g) continue;
        for (int ty = 0; ty < tiles_y; ++ty) {
            int cy0, ny;
            tile_nodes(ty * TS, GY, H, cy0, ny);
            if (cy0 > y) break;                      // the first node grows with the tile index
            if (y >= cy0 + ny) continue;
            for (int tx = 0; tx < tiles_x; ++tx) {
                int cx0, nx;
                tile_nodes(tx * TS, GX, W, cx0, nx);
                if (cx0 > x) break;
                if (x >= cx0 + nx) continue;
                const float* p = partials + (((size_t)v * tiles_y + ty) * tiles_x + tx) * slab;
                sum = add_(sum, p[((n * ny + (y - cy0)) * nx + (x - cx0)) * 12 + k]);
            }
        }
    }
    dgrids[e] = sum;
}

size_t slab_floats(const Shape& s) { return s.nodes() * 12; }
size_t fwd_smem(const Shape& s) { return s.nodes() * 12 * sizeof(float); }
size_t bwd_smem(const Shape& s, bool grid) {
    return s.nodes() * 12 * sizeof(float) * (grid ? 2 : 1) + (grid ? TS * sizeof(PixRec) : 0);
}

template <typename K>
int set_smem(K kernel, size_t bytes) {
    if (bytes > 48 * 1024) R3DG_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return 0;
}

template <int R, bool GRID>
int launch_bwd(const Shape& s, const float* grids, const int* ids, const float* rgb, const float* dout, float* drgb,
               float* partials, cudaStream_t stream) {
    auto kernel = bilagrid_bwd_kernel<R, GRID>;
    const size_t smem = bwd_smem(s, GRID);
    if (const int rc = set_smem(kernel, smem)) return rc;
    kernel<<<dim3(s.tiles_x(), s.tiles_y(), s.N), 32, smem, stream>>>(s.H, s.W, s.GX, s.GY, s.L, (int)slab_floats(s),
                                                                     grids, ids, rgb, dout, drgb, partials);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace

size_t bilagrid_tmp_bytes(int G, int N, int H, int W, int GX, int GY, int L) {
    Shape s;
    if (check(G, N, H, W, GX, GY, L, s) != 0) return 0;
    return align_up((size_t)s.tiles_x() * s.tiles_y() * N * slab_floats(s) * sizeof(float), 256);
}

int launch_bilagrid_forward(int G, int N, int H, int W, int GX, int GY, int L, const float* grids, const int* ids,
                            const float* rgb, float* out, cudaStream_t stream) {
    Shape s;
    const int rc = check(G, N, H, W, GX, GY, L, s);
    if (rc != 0) return rc;
    if (!grids || !ids || !rgb || !out) return R3DG_ERR_BAD_ARG;
    const size_t smem = fwd_smem(s);
    if (const int e = set_smem(bilagrid_fwd_kernel, smem)) return e;
    bilagrid_fwd_kernel<<<dim3(s.tiles_x(), s.tiles_y(), N), FWD_NT, smem, stream>>>(H, W, GX, GY, L, grids, ids, rgb, out);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_bilagrid_backward(int G, int N, int H, int W, int GX, int GY, int L, const float* grids, const int* ids,
                             const float* rgb, const float* dL_dout, float* dL_drgb, float* dL_dgrids, void* tmp,
                             size_t tmp_bytes, cudaStream_t stream) {
    Shape s;
    const int rc = check(G, N, H, W, GX, GY, L, s);
    if (rc != 0) return rc;
    if (!grids || !ids || !rgb || !dL_dout || (!dL_drgb && !dL_dgrids)) return R3DG_ERR_BAD_ARG;
    if (dL_dgrids && (!tmp || tmp_bytes < bilagrid_tmp_bytes(G, N, H, W, GX, GY, L))) return R3DG_ERR_BAD_ARG;
    const bool two = 4 * L > 32;
    float* part = static_cast<float*>(tmp);
    int e;
    if (!dL_dgrids) e = two ? launch_bwd<2, false>(s, grids, ids, rgb, dL_dout, dL_drgb, nullptr, stream)
                            : launch_bwd<1, false>(s, grids, ids, rgb, dL_dout, dL_drgb, nullptr, stream);
    else e = two ? launch_bwd<2, true>(s, grids, ids, rgb, dL_dout, dL_drgb, part, stream)
                 : launch_bwd<1, true>(s, grids, ids, rgb, dL_dout, dL_drgb, part, stream);
    if (e != 0) return e;
    if (dL_dgrids) {
        const long long total = (long long)G * 12 * L * GY * GX;
        bilagrid_reduce_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(G, N, H, W, GX, GY, L,
                                                                                 (int)slab_floats(s), ids, part,
                                                                                 dL_dgrids);
        R3DG_CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

}  // namespace r3dg
