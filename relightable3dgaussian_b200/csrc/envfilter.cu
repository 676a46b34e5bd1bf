// The lat-long mip pyramid of the shading step's filtered mode (include/r3dg_b200.h, "PREFILTERED ENVIRONMENT"):
// its build, one launch per coarser level, and the adjoint the shading backward folds into dL/denv, two launches per
// coarser level.  Both are gathers in a fixed order with fp64 sums and no atomics, so they are bitwise reproducible.
//
// The stencil is an area-weighted box filter on the sphere.  Row j of an h-row level stands for the latitude band
// [(j - 1/2) dt, (j + 1/2) dt] clipped to [0, pi] (dt = pi / (h - 1): rows 0 and h - 1 are the polar caps), column i of
// a w-column level for the azimuth cell [(i - 1/2) dp, (i + 1/2) dp] with dp = 2 pi / (w - 1), modulo 2 pi (columns 0
// and w - 1 are the same cell).  A texel's weight is the solid angle of its cell, cos(top) - cos(bottom) times the
// cell's azimuth: 2 sin(dt / 2) dp sin(theta_j) inside, (1 - cos(dt / 2)) dp at a pole, i.e. sin(theta) clamped at the
// pole rows.  A coarse texel is the mean of the finer level over its cell, each finer texel weighted by the solid angle
// its cell shares with the coarse one; the pole rows average the whole cap, and the last column repeats column 0.
// The coarse cells tile the sphere as the fine ones do, so the solid-angle-weighted mean is kept at every level; the
// weights are normalised by their own sum, so a constant env stays that constant exactly.
#include "common.cuh"
#include "envfilter.cuh"
#include "kernels.h"

namespace r3dg {

#define EF_THREADS 256
#define EF_PI 3.14159265358979323846

// solid angle per radian of azimuth shared by row j of an h-row level and row k of an h2-row level
__device__ __forceinline__ double band_overlap(int j, int h, int k, int h2) {
    const double d = EF_PI / (h - 1), d2 = EF_PI / (h2 - 1);
    const double lo = fmax(fmax((j - 0.5) * d, (k - 0.5) * d2), 0.0);
    const double hi = fmin(fmin((j + 0.5) * d, (k + 0.5) * d2), EF_PI);
    return hi > lo ? cos(lo) - cos(hi) : 0.0;
}

// azimuth shared by the cell at unwrapped position m of a w-column level and cell i of a w2-column level
__device__ __forceinline__ double cell_overlap(int m, int w, int i, int w2) {
    const double d = 2.0 * EF_PI / (w - 1), d2 = 2.0 * EF_PI / (w2 - 1);
    const double lo = fmax((m - 0.5) * d, (i - 0.5) * d2), hi = fmin((m + 0.5) * d, (i + 0.5) * d2);
    return hi > lo ? hi - lo : 0.0;
}

// the cells of an n-cell grid (spacing d) that may overlap cell k of spacing d2: [lo, hi]
__device__ __forceinline__ void cover(int k, double d2, double d, int& lo, int& hi) {
    lo = (int)floor((k - 0.5) * d2 / d - 0.5);
    hi = (int)ceil((k + 0.5) * d2 / d + 0.5);
}

__device__ __forceinline__ int wrap(int m, int n) { return ((m % n) + n) % n; }

// sum of the row weights of coarse row k (the forward's normaliser, in its order)
__device__ __forceinline__ double row_weight(int k, int h2, int h) {
    int lo, hi;
    cover(k, EF_PI / (h2 - 1), EF_PI / (h - 1), lo, hi);
    double s = 0.0;
    for (int j = max(lo, 0); j <= min(hi, h - 1); ++j) s += band_overlap(j, h, k, h2);
    return s;
}

// sum of the column weights of coarse column i (< w2 - 1)
__device__ __forceinline__ double col_weight(int i, int w2, int w) {
    int lo, hi;
    cover(i, 2.0 * EF_PI / (w2 - 1), 2.0 * EF_PI / (w - 1), lo, hi);
    double s = 0.0;
    for (int m = lo; m <= hi; ++m) s += cell_overlap(m, w, i, w2);
    return s;
}

// fixed-order block sum of three doubles per thread; the totals are valid in every thread
__device__ __forceinline__ void block_sum3(double* v, double (*red)[EF_THREADS]) {
    for (int c = 0; c < 3; ++c) red[c][threadIdx.x] = v[c];
    __syncthreads();
    for (int s = EF_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s)
            for (int c = 0; c < 3; ++c) red[c][threadIdx.x] += red[c][threadIdx.x + s];
        __syncthreads();
    }
    for (int c = 0; c < 3; ++c) v[c] = red[c][0];
    __syncthreads();
}

// coarse [h2,w2,3] from fine [h,w,3]: blocks 0 and 1 write the two pole rows, the others one interior texel per thread
__global__ void __launch_bounds__(EF_THREADS) env_down_kernel(const float* __restrict__ fine, int h, int w,
                                                              float* __restrict__ coarse, int h2, int w2) {
    if (blockIdx.x < 2) {
        __shared__ double red[3][EF_THREADS];
        const int k = blockIdx.x == 0 ? 0 : h2 - 1;
        int lo, hi;
        cover(k, EF_PI / (h2 - 1), EF_PI / (h - 1), lo, hi);
        double acc[3] = {0.0, 0.0, 0.0}, wsum = 0.0;
        for (int j = max(lo, 0); j <= min(hi, h - 1); ++j) {
            const double a = band_overlap(j, h, k, h2);
            if (a == 0.0) continue;                      // uniform over the block
            double s[3] = {0.0, 0.0, 0.0};
            for (int m = threadIdx.x; m < w - 1; m += EF_THREADS)
                for (int c = 0; c < 3; ++c) s[c] += fine[((size_t)j * w + m) * 3 + c];
            block_sum3(s, red);
            for (int c = 0; c < 3; ++c) acc[c] += a * (s[c] / (w - 1));
            wsum += a;
        }
        for (int i = threadIdx.x; i < w2; i += EF_THREADS)
            for (int c = 0; c < 3; ++c) coarse[((size_t)k * w2 + i) * 3 + c] = (float)(acc[c] / wsum);
        return;
    }
    const long long t = (long long)(blockIdx.x - 2) * EF_THREADS + threadIdx.x;
    if (t >= (long long)(h2 - 2) * w2) return;
    const int k = 1 + (int)(t / w2), i = (int)(t % w2);
    const int ic = i == w2 - 1 ? 0 : i;                  // the seam column repeats column 0
    int jlo, jhi, mlo, mhi;
    cover(k, EF_PI / (h2 - 1), EF_PI / (h - 1), jlo, jhi);
    cover(ic, 2.0 * EF_PI / (w2 - 1), 2.0 * EF_PI / (w - 1), mlo, mhi);
    double num[3] = {0.0, 0.0, 0.0};
    for (int j = max(jlo, 0); j <= min(jhi, h - 1); ++j) {
        const double a = band_overlap(j, h, k, h2);
        if (a == 0.0) continue;
        double r[3] = {0.0, 0.0, 0.0};
        for (int m = mlo; m <= mhi; ++m) {
            const double b = cell_overlap(m, w, ic, w2);
            if (b == 0.0) continue;
            const float* f = fine + ((size_t)j * w + wrap(m, w - 1)) * 3;
            for (int c = 0; c < 3; ++c) r[c] += b * (double)f[c];
        }
        for (int c = 0; c < 3; ++c) num[c] += a * r[c];
    }
    const double den = row_weight(k, h2, h) * col_weight(ic, w2, w);
    for (int c = 0; c < 3; ++c) coarse[((size_t)k * w2 + i) * 3 + c] = (float)(num[c] / den);
}

// adjoint, step 1: the gradient of each pole row of the coarse level [h2,w2,3], summed over its columns (every column
// of a pole row is the same cap average), into column 0 of that row
__global__ void __launch_bounds__(EF_THREADS) env_pole_fold_kernel(float* __restrict__ g2, int h2, int w2) {
    __shared__ double red[3][EF_THREADS];
    const int k = blockIdx.x == 0 ? 0 : h2 - 1;
    double s[3] = {0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < w2; i += EF_THREADS)
        for (int c = 0; c < 3; ++c) s[c] += g2[((size_t)k * w2 + i) * 3 + c];
    block_sum3(s, red);
    if (threadIdx.x == 0)
        for (int c = 0; c < 3; ++c) g2[(size_t)k * w2 * 3 + c] = (float)s[c];
}

// adjoint, step 2: out[f] = g[f] + sum over the coarse texels k that read fine texel f of weight(k, f) g2[k], one fine
// texel [h,w,3] per thread (out may be g)
__global__ void __launch_bounds__(EF_THREADS) env_up_kernel(const float* g, int h, int w, const float* __restrict__ g2,
                                                            int h2, int w2, float* out) {
    const long long t = (long long)blockIdx.x * EF_THREADS + threadIdx.x;
    if (t >= (long long)h * w) return;
    const int j = (int)(t / w), m = (int)(t % w);
    double acc[3] = {0.0, 0.0, 0.0};
    if (m < w - 1) {                                     // the fine seam column is not read by the coarser level
        int klo, khi;
        cover(j, EF_PI / (h - 1), EF_PI / (h2 - 1), klo, khi);
        for (int k = max(klo, 0); k <= min(khi, h2 - 1); ++k) {
            const double a = band_overlap(j, h, k, h2);
            if (a == 0.0) continue;
            const double rw = row_weight(k, h2, h);
            if (k == 0 || k == h2 - 1) {                 // a cap: the folded row total, spread over the fine columns
                const float* G = g2 + (size_t)k * w2 * 3;
                for (int c = 0; c < 3; ++c) acc[c] += a / (rw * (w - 1)) * (double)G[c];
                continue;
            }
            for (int shift = -(w - 1); shift <= w - 1; shift += w - 1) {
                const int mm = m + shift;
                int ilo, ihi;
                cover(mm, 2.0 * EF_PI / (w - 1), 2.0 * EF_PI / (w2 - 1), ilo, ihi);
                for (int i = max(ilo, 0); i <= min(ihi, w2 - 2); ++i) {
                    const double b = cell_overlap(mm, w, i, w2);
                    if (b == 0.0) continue;
                    const float* G = g2 + ((size_t)k * w2 + i) * 3;
                    const float* Gs = g2 + ((size_t)k * w2 + w2 - 1) * 3;      // the seam column reads column 0's cell
                    const double wt = a * b / (rw * col_weight(i, w2, w));
                    for (int c = 0; c < 3; ++c) acc[c] += wt * ((double)G[c] + (i == 0 ? (double)Gs[c] : 0.0));
                }
            }
        }
    }
    for (int c = 0; c < 3; ++c) out[(size_t)t * 3 + c] = (float)((double)g[(size_t)t * 3 + c] + acc[c]);
}

static unsigned ef_blocks(long long n) { return (unsigned)((n + EF_THREADS - 1) / EF_THREADS); }

int launch_env_pyramid_adjoint(const EnvLevels& lv, float* g, float* d_env, cudaStream_t stream) {
    if (lv.L == 1) {
        R3DG_CUDA_TRY(cudaMemcpyAsync(d_env, g, (size_t)lv.h[0] * lv.w[0] * 3 * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return 0;
    }
    for (int l = lv.L - 2; l >= 0; --l) {
        float* fine = g + (size_t)lv.off[l] * 3;
        float* coarse = g + (size_t)lv.off[l + 1] * 3;
        env_pole_fold_kernel<<<2, EF_THREADS, 0, stream>>>(coarse, lv.h[l + 1], lv.w[l + 1]);
        R3DG_CUDA_TRY(cudaGetLastError());
        env_up_kernel<<<ef_blocks((long long)lv.h[l] * lv.w[l]), EF_THREADS, 0, stream>>>(
            fine, lv.h[l], lv.w[l], coarse, lv.h[l + 1], lv.w[l + 1], l == 0 ? d_env : fine);
        R3DG_CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

}  // namespace r3dg

// ---- C ABI --------------------------------------------------------------------------------------
using namespace r3dg;
extern "C" {

int r3dg_env_pyramid_levels(int env_h, int env_w) { return env_h > 0 && env_w > 0 ? env_levels(env_h, env_w).L : 0; }

size_t r3dg_env_pyramid_floats(int env_h, int env_w) {
    return env_h > 0 && env_w > 0 ? (size_t)env_levels(env_h, env_w).total * 3 : 0;
}

int r3dg_env_pyramid_build(const float* env, int env_h, int env_w, float* pyramid, r3dg_stream_t stream) {
    if (!env || !pyramid || env_h <= 0 || env_w <= 0) return R3DG_ERR_BAD_ARG;
    const EnvLevels lv = env_levels(env_h, env_w);
    const cudaStream_t s = (cudaStream_t)stream;
    R3DG_CUDA_TRY(cudaMemcpyAsync(pyramid, env, (size_t)env_h * env_w * 3 * sizeof(float), cudaMemcpyDeviceToDevice, s));
    for (int l = 1; l < lv.L; ++l) {
        env_down_kernel<<<2 + ef_blocks((long long)(lv.h[l] - 2) * lv.w[l]), EF_THREADS, 0, s>>>(
            pyramid + (size_t)lv.off[l - 1] * 3, lv.h[l - 1], lv.w[l - 1], pyramid + (size_t)lv.off[l] * 3, lv.h[l], lv.w[l]);
        R3DG_CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

}  // extern "C"
