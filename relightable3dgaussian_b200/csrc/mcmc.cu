// MCMC densification (3DGS-MCMC, Kheradmand et al. 2024; gsplat's MCMCStrategy): relocation of dead Gaussians onto
// live ones and growth under a budget, plus the per-step position noise.  The host side is relightable3dgaussian_b200/
// mcmc.py.  Every kernel is HBM-bound except the fp64 source update, which runs on the few sampled rows only.
//   mcmc_noise_kernel     xyz += scale sigma(-k (o - t)) Sigma z, one thread per row, in place, in fp64;
//   mcmc_classify_kernel  per row: weight, alive flag, zeroed draw count; per block: the fp64 sum of the weights;
//   mcmc_scan_kernel      exclusive fp64 scan of the block sums (one CTA, fixed order);
//   mcmc_cdf_kernel       the inclusive fp64 CDF of the weights (classify's block scan again, plus the block prefix);
//   mcmc_draw_kernel      inverse-CDF draws, one per uniform; integer atomics count the draws of each source;
//   mcmc_update_kernel    the opacity / scale correction of every drawn source, in fp64, into tmp;
//   mcmc_apply_kernel     every tensor written once from the old one (descriptor table, one blockIdx.y per tensor).
// The weights are summed in a fixed order (per thread, then a warp-shuffle scan, then the block scan of scan_kernel),
// so repeated calls are bitwise equal; the draws land on sources by integer atomics only.
#include "common.cuh"
#include "kernels.h"

namespace r3dg {

#define MC_THREADS 256
#define MC_ITEMS 8
#define MC_TILE (MC_THREADS * MC_ITEMS)

// tmp layout, every region 256-byte aligned; only the last one depends on n_new, so classify (sized for n_new = 0) and
// apply see the same offsets
struct McmcTmp {
    size_t cdf, bsum, weight, count, pick, alive, newv, total;
    long long nblocks;
    __host__ McmcTmp(int P, int n_new) {
        nblocks = ((long long)P + MC_TILE - 1) / MC_TILE;
        const size_t rows = (size_t)(P < 1 ? 1 : P);
        const size_t draws = (size_t)(n_new > P ? n_new : P < 1 ? 1 : P);
        size_t off = 0;
        cdf = off;   off = align_up(off + rows * 8, 256);                    // double [P]  inclusive CDF
        bsum = off;  off = align_up(off + (size_t)(nblocks + 1) * 8, 256);   // double [nblocks]  block sums -> exclusive prefix
        weight = off; off = align_up(off + rows * 4, 256);                   // float [P]  sampling weights
        count = off; off = align_up(off + rows * 4, 256);                    // u32 [P]  draws per source
        alive = off; off = align_up(off + rows, 256);                        // u8 [P]
        newv = off;  off = align_up(off + rows * 16, 256);                   // float4 [P]  (l', s'0, s'1, s'2) of each source
        pick = off;  off = align_up(off + draws * 4, 256);                   // int [max(P, n_new)]  source of each draw or -1
        total = off;
    }
};

// torch's CUDA fp32 sigmoid 1 / (1 + expf(-x)): the IEEE quotient 1 / d is the correctly rounded reciprocal of d
__device__ __forceinline__ float sigmoid32(float x) { return __frcp_rn(__fadd_rn(1.f, expf(-x))); }

// Evaluated in fp64 and rounded once: the gate's argument -k (o - t) reaches -100, where an fp32 difference would cost
// ~|a| eps32 of relative accuracy, and an fp32 rotation matrix has absolute errors that a strongly anisotropic
// covariance does not scale down.  The fp64 work (~100 operations a row) stays under the kernel's HBM time.
__global__ void __launch_bounds__(256) mcmc_noise_kernel(int P, float* __restrict__ xyz, const float* __restrict__ rot,
                                                         const float* __restrict__ scl, const float* __restrict__ opac,
                                                         const float* __restrict__ z, double scale, double k, double t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const double o = (double)sigmoid32(opac[i]);
    const double g = scale / (1.0 + exp(k * (o - t)));
    // scalar loads: a contiguous [P,4] tensor need not be 16-byte aligned (a row slice of a larger one)
    const double qr = rot[4LL * i], qx = rot[4LL * i + 1], qy = rot[4LL * i + 2], qz = rot[4LL * i + 3];
    const double inv = 1.0 / sqrt(qr * qr + qx * qx + qy * qy + qz * qz);
    const double r = qr * inv, x = qx * inv, y = qy * inv, w = qz * inv;
    const double R[3][3] = {{1.0 - 2.0 * (y * y + w * w), 2.0 * (x * y - r * w), 2.0 * (x * w + r * y)},
                            {2.0 * (x * y + r * w), 1.0 - 2.0 * (x * x + w * w), 2.0 * (y * w - r * x)},
                            {2.0 * (x * w - r * y), 2.0 * (y * w + r * x), 1.0 - 2.0 * (x * x + y * y)}};
    double e2[3], zr[3], v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        e2[c] = exp(2.0 * (double)scl[3LL * i + c]);
        zr[c] = z[3LL * i + c];
    }
    // Sigma z = R diag(e^2) (R^T z)
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = e2[c] * (R[0][c] * zr[0] + R[1][c] * zr[1] + R[2][c] * zr[2]);
#pragma unroll
    for (int c = 0; c < 3; ++c)
        xyz[3LL * i + c] = (float)((double)xyz[3LL * i + c] + g * (R[c][0] * v[0] + R[c][1] * v[1] + R[c][2] * v[2]));
}

// Block scan of the weights of one tile of MC_TILE rows: thread t owns MC_ITEMS consecutive rows, with weights w.
// incl[k] gets the inclusive prefix within the block of the thread's row k; the return value is the block total (the
// last prefix).  classify and cdf both call it on the same weights, so the block sums and the CDF agree bit for bit.
__device__ __forceinline__ double block_scan_weights(const float (&w)[MC_ITEMS], double (&incl)[MC_ITEMS]) {
    __shared__ double s_warp[MC_THREADS / 32];
    __shared__ double s_total;
    double run = 0.0;
#pragma unroll
    for (int k = 0; k < MC_ITEMS; ++k) {
        run += (double)w[k];
        incl[k] = run;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double inc = run;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) { const double v = __shfl_up_sync(0xffffffffu, inc, s); if (lane >= s) inc += v; }
    double ex = __shfl_up_sync(0xffffffffu, inc, 1);   // exclusive prefix within the warp
    if (lane == 0) ex = 0.0;
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    double pre = 0.0;
    for (int i = 0; i < warp; ++i) pre += s_warp[i];
    pre += ex;                                         // exclusive prefix of this thread within the block
    if (threadIdx.x == MC_THREADS - 1) s_total = pre + run;
#pragma unroll
    for (int k = 0; k < MC_ITEMS; ++k) incl[k] += pre;
    __syncthreads();
    return s_total;
}

// Weights (0 for dead rows) and alive flags to tmp, draw counts zeroed, block sums.  cdf reads the weights back instead
// of evaluating the sigmoid again: its IEEE reciprocal has an out-of-line slow path, and that call would make the fp64
// scan there spill.
__global__ void __launch_bounds__(MC_THREADS) mcmc_classify_kernel(int P, const float* __restrict__ opac, float min_opacity,
                                                                   float* __restrict__ weight, double* __restrict__ bsum,
                                                                   uint32_t* __restrict__ count, uint8_t* __restrict__ alive) {
    const long long row0 = (long long)blockIdx.x * MC_TILE + (long long)threadIdx.x * MC_ITEMS;
    float w[MC_ITEMS];
#pragma unroll
    for (int k = 0; k < MC_ITEMS; ++k) {
        w[k] = 0.f;
        if (row0 + k < P) {
            const float o = sigmoid32(opac[row0 + k]);
            const bool a = o > min_opacity;
            w[k] = a ? o : 0.f;
            weight[row0 + k] = w[k];
            alive[row0 + k] = a;
            count[row0 + k] = 0u;
        }
    }
    double incl[MC_ITEMS];
    const double tot = block_scan_weights(w, incl);
    if (threadIdx.x == 0) bsum[blockIdx.x] = tot;
}

// Exclusive scan of the n block sums in place, in 1024-element chunks carried in order.  One CTA of 1024 threads.
__global__ void __launch_bounds__(1024) mcmc_scan_kernel(long long n, double* __restrict__ bsum) {
    __shared__ double s_warp[32];
    __shared__ double s_carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0.0;
    __syncthreads();
    for (long long base = 0; base < n; base += 1024) {
        const long long i = base + threadIdx.x;
        const double v = i < n ? bsum[i] : 0.0;
        double inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const double t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        double ex = __shfl_up_sync(0xffffffffu, inc, 1);
        if (lane == 0) ex = 0.0;
        if (lane == 31) s_warp[warp] = inc;
        __syncthreads();
        if (warp == 0) {
            double winc = s_warp[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const double t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
            double wex = __shfl_up_sync(0xffffffffu, winc, 1);
            s_warp[lane] = lane == 0 ? 0.0 : wex;                // exclusive prefix of the warp totals
        }
        __syncthreads();
        const double excl = s_carry + (s_warp[warp] + ex);
        if (i < n) bsum[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = excl + v;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(MC_THREADS) mcmc_cdf_kernel(int P, const float* __restrict__ weight,
                                                              const double* __restrict__ bexcl, double* __restrict__ cdf) {
    const long long row0 = (long long)blockIdx.x * MC_TILE + (long long)threadIdx.x * MC_ITEMS;
    float w[MC_ITEMS];
#pragma unroll
    for (int k = 0; k < MC_ITEMS; ++k) w[k] = row0 + k < P ? weight[row0 + k] : 0.f;
    double incl[MC_ITEMS];
    block_scan_weights(w, incl);
    const double pre = bexcl[blockIdx.x];
#pragma unroll
    for (int k = 0; k < MC_ITEMS; ++k)
        if (row0 + k < P) cdf[row0 + k] = pre + incl[k];
}

// Draw d picks the smallest i with cdf[i] > u_d * total.  With no live row (total 0) every row weighs 1: i = floor(u_d P).
// Relocation (grow == 0): draw d belongs to row d and only dead rows draw, and only when a live row exists.
// The CDF is monotone only up to rounding: where two partial sums meet (every 8-row thread boundary, every block
// boundary) a prefix can round one ulp above or below the value before it.  A target inside such a one-ulp step can
// land on a zero-weight row; the search then moves to the next live row (the previous one at the end).  So a dead row
// is never a source, and relocation never reads a row it rewrites.
__global__ void __launch_bounds__(256) mcmc_draw_kernel(int P, long long ndraw, int grow, const float* __restrict__ u,
                                                        const double* __restrict__ cdf, const uint8_t* __restrict__ alive,
                                                        int* __restrict__ pick, uint32_t* __restrict__ count) {
    const long long d = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= ndraw) return;
    const double total = cdf[P - 1];
    int src = -1;
    if (grow || (!alive[d] && total > 0.0)) {
        if (total > 0.0) {
            const double v = (double)u[d] * total;
            int lo = 0, hi = P - 1;
            while (lo < hi) {
                const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
                if (cdf[mid] > v) hi = mid; else lo = mid + 1;
            }
            if (!alive[lo]) {
                int i = lo;
                while (i < P - 1 && !alive[i]) ++i;
                if (!alive[i])
                    for (i = lo; i > 0 && !alive[i]; --i) {}
                lo = i;
            }
            src = lo;
        } else {
            src = (int)min((double)(P - 1), floor((double)u[d] * (double)P));
        }
        atomicAdd(count + src, 1u);
    }
    pick[d] = src;
}

// Binomial coefficients C(n, j), n <= R3DG_MCMC_MAX_N, rounded once from the exact integers (exact up to n = 56).
struct BinomTable {
    double c[R3DG_MCMC_MAX_N + 1][R3DG_MCMC_MAX_N + 1];
    constexpr BinomTable() : c() {
        unsigned long long row[R3DG_MCMC_MAX_N + 1] = {};
        row[0] = 1;
        for (int n = 0; n <= R3DG_MCMC_MAX_N; ++n) {
            if (n > 0)
                for (int j = n; j > 0; --j) row[j] += row[j - 1];
            for (int j = 0; j <= n; ++j) c[n][j] = (double)row[j];
        }
    }
};
__constant__ BinomTable kBinom = BinomTable();

// Source i drawn c >= 1 times: N = min(c + 1, n_max), o = sigma32(l) in fp64, x = 1 - (1 - o)^(1/N),
// coef = o / sum_{j=1..N} (-1)^(j-1) C(N,j) x^j / sqrt(j), l' = logit(clamp(x, min_opacity, 1 - 2^-23)),
// s' = s + log coef.  x is evaluated as -expm1(log1p(-o) / N), accurate for every o; o = 0 (fp32 underflow) gives
// x = 0, where coef takes its limit 1.
__global__ void __launch_bounds__(256) mcmc_update_kernel(int P, const float* __restrict__ opac, const float* __restrict__ scl,
                                                          const uint32_t* __restrict__ count, double min_opacity, int n_max,
                                                          float4* __restrict__ newv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const uint32_t c = count[i];
    if (c == 0) return;
    const int N = (int)min((unsigned long long)c + 1ull, (unsigned long long)n_max);
    const double o = (double)sigmoid32(opac[i]);
    const double x = -expm1(log1p(-o) / (double)N);
    double coef = 1.0;
    if (x > 0.0) {
        double sum = 0.0, xp = 1.0;
        for (int j = 1; j <= N; ++j) {
            xp = __dmul_rn(xp, x);
            const double term = __ddiv_rn(__dmul_rn(kBinom.c[N][j], xp), sqrt((double)j));
            sum = (j & 1) ? __dadd_rn(sum, term) : __dsub_rn(sum, term);
        }
        coef = o / sum;
    }
    const double on = fmin(fmax(x, min_opacity), 1.0 - 0x1p-23);
    const double lc = log(coef);
    newv[i] = make_float4((float)log(on / (1.0 - on)), (float)((double)scl[3LL * i] + lc),
                          (float)((double)scl[3LL * i + 1] + lc), (float)((double)scl[3LL * i + 2] + lc));
}

struct McmcApplyParams {
    long long P, Pn;            // input rows, output rows (P in place, P + n_new grown)
    int grow;
    const int* pick;
    const uint32_t* count;
    const float4* newv;
    int num;
    r3dg_densify_tensor t[R3DG_DENSIFY_MAX];
};

// Output row r takes the values of row `from`: r itself, the source a dead row drew (relocation), or the source of
// growth draw r - P.  A rewritten row (a drawn source or a copy of one) gets the corrected opacity / scale and zero
// moments and statistics.  In place (relocation) only rewritten rows are written.
__global__ void __launch_bounds__(256) mcmc_apply_kernel(const McmcApplyParams p) {
    const r3dg_densify_tensor t = p.t[blockIdx.y];
    const long long wpr = t.row_bytes >> 2;
    const uint32_t* src = (const uint32_t*)t.src;
    uint32_t* dst = (uint32_t*)t.dst;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const bool narrow = p.Pn * wpr < (1LL << 32);          // 32-bit division is several times cheaper than 64-bit
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < p.Pn * wpr; j += stride) {
        const long long r = narrow ? (long long)((uint32_t)j / (uint32_t)wpr) : j / wpr;
        const int w = (int)(j - r * wpr);
        long long from = r;
        bool rewritten;
        if (r >= p.P) {
            from = p.pick[r - p.P];
            rewritten = true;
        } else if (!p.grow && p.pick[r] >= 0) {
            from = p.pick[r];
            rewritten = true;
        } else {
            rewritten = p.count[r] != 0u;
        }
        if (!p.grow && (!rewritten || (from == r && t.kind == R3DG_DENSIFY_COPY))) continue;
        uint32_t v;
        if (rewritten && t.kind == R3DG_DENSIFY_MOMENT) v = 0u;
        else if (rewritten && t.kind == R3DG_MCMC_OPACITY) v = __float_as_uint(p.newv[from].x);
        else if (rewritten && t.kind == R3DG_MCMC_SCALING) v = __float_as_uint((&p.newv[from].y)[w]);
        else v = src[from * wpr + w];
        dst[j] = v;
    }
}

size_t mcmc_tmp_bytes(int P, int n_new) { return McmcTmp(P, n_new).total; }

int launch_mcmc_noise(int P, float* xyz, const float* rotation, const float* scaling, const float* opacity, const float* z,
                      double scale, double k, double t, cudaStream_t stream) {
    if (P < 0) return R3DG_ERR_BAD_ARG;
    if (P == 0) return 0;
    if (!xyz || !rotation || !scaling || !opacity || !z) return R3DG_ERR_BAD_ARG;
    mcmc_noise_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, xyz, rotation, scaling, opacity, z, scale, k, t);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_mcmc_classify(int P, const float* opacity, float min_opacity, void* tmp_, size_t tmp_bytes, cudaStream_t stream) {
    const McmcTmp t(P, 0);
    if (P <= 0 || !opacity || !tmp_ || ((uintptr_t)tmp_ & 15) || tmp_bytes < t.total) return R3DG_ERR_BAD_ARG;
    char* tmp = (char*)tmp_;
    double* bsum = (double*)(tmp + t.bsum);
    float* weight = (float*)(tmp + t.weight);
    mcmc_classify_kernel<<<(unsigned)t.nblocks, MC_THREADS, 0, stream>>>(P, opacity, min_opacity, weight, bsum,
                                                                         (uint32_t*)(tmp + t.count), (uint8_t*)(tmp + t.alive));
    mcmc_scan_kernel<<<1, 1024, 0, stream>>>(t.nblocks, bsum);
    mcmc_cdf_kernel<<<(unsigned)t.nblocks, MC_THREADS, 0, stream>>>(P, weight, bsum, (double*)(tmp + t.cdf));
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_mcmc_apply(int P, int n_new, const float* u, const float* opacity, const float* scaling, double min_opacity, int n_max,
                      int num, const r3dg_densify_tensor* tensors, void* tmp_, size_t tmp_bytes, int num_sms,
                      cudaStream_t stream) {
    const McmcTmp t(P, n_new);
    if (P <= 0 || n_new < 0 || (long long)P + n_new > 0x7fffffffLL || !u || !opacity || !scaling || n_max < 2 ||
        n_max > R3DG_MCMC_MAX_N || num < 1 || num > R3DG_DENSIFY_MAX || !tensors || !tmp_ || ((uintptr_t)tmp_ & 15) || tmp_bytes < t.total)
        return R3DG_ERR_BAD_ARG;
    const bool grow = n_new > 0;
    McmcApplyParams p;
    p.P = P; p.Pn = (long long)P + n_new; p.grow = grow ? 1 : 0; p.num = num;
    char* tmp = (char*)tmp_;
    p.pick = (const int*)(tmp + t.pick);
    p.count = (const uint32_t*)(tmp + t.count);
    p.newv = (const float4*)(tmp + t.newv);
    for (int k = 0; k < num; ++k) {
        const r3dg_densify_tensor& d = tensors[k];
        const bool kind_ok = d.kind == R3DG_DENSIFY_COPY || d.kind == R3DG_DENSIFY_MOMENT || d.kind == R3DG_MCMC_OPACITY ||
                             d.kind == R3DG_MCMC_SCALING;
        if (!kind_ok || d.row_bytes <= 0 || (d.row_bytes & 3) || !d.src || !d.dst) return R3DG_ERR_BAD_ARG;
        if ((grow && d.src == d.dst) || (!grow && d.src != d.dst)) return R3DG_ERR_BAD_ARG;
        if ((d.kind == R3DG_MCMC_OPACITY && d.row_bytes != 4) || (d.kind == R3DG_MCMC_SCALING && d.row_bytes != 12))
            return R3DG_ERR_BAD_ARG;
        p.t[k] = d;
    }
    const long long ndraw = grow ? n_new : P;
    mcmc_draw_kernel<<<(unsigned)((ndraw + 255) / 256), 256, 0, stream>>>(P, ndraw, p.grow, u, (const double*)(tmp + t.cdf),
                                                                          (const uint8_t*)(tmp + t.alive), (int*)(tmp + t.pick),
                                                                          (uint32_t*)(tmp + t.count));
    mcmc_update_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, opacity, scaling, (const uint32_t*)(tmp + t.count), min_opacity,
                                                            n_max, (float4*)(tmp + t.newv));
    mcmc_apply_kernel<<<dim3((unsigned)(num_sms * 8), (unsigned)num), 256, 0, stream>>>(p);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
