// Importance sampling of the environment light (include/r3dg_b200.h, IMPORTANCE SAMPLING; DESIGN.md §4.31): the env
// table's build and the per-row sampler whose directions and areas feed the unchanged trace and shading step.
// Compiled with the default flags; the sampler's arithmetic (importance.cuh) is rounded op by op, so any kernel that
// includes it reproduces these bits.
#include "importance.cuh"

namespace r3dg {

#define IS_BUILD_THREADS 256

// the cell geometry of the env-filter stencil: row j is the band [(j - 1/2) dt, (j + 1/2) dt] clipped to [0, pi]
__device__ __forceinline__ double band_lo(int j, int He) { return fmax((j - 0.5) * (M_PI / (He - 1)), 0.0); }
__device__ __forceinline__ double band_hi(int j, int He) { return fmin((j + 0.5) * (M_PI / (He - 1)), M_PI); }
__device__ __forceinline__ double cell_solid_angle(int j, int He, int We) {
    return (cos(band_lo(j, He)) - cos(band_hi(j, He))) * (2.0 * M_PI / (We - 1));
}

// max(lum, 0) over the 3 x 3 texels around cell (j, i): rows clamped, columns wrapped over the We - 1 distinct azimuths
// (texel column We - 1 is azimuth 0); a non-finite luminance counts as 0
__device__ __forceinline__ double cell_max_lum(const float* __restrict__ env, int He, int We, int j, int i) {
    double m = 0.0;
    const int C = We - 1;
    for (int dj = -1; dj <= 1; ++dj) {
        const int jj = min(max(j + dj, 0), He - 1);
        for (int di = -1; di <= 1; ++di) {
            const int c = ((i + di) % C + C) % C;
            for (int rep = 0; rep < (c == 0 ? 2 : 1); ++rep) {
                const float* p = env + ((size_t)jj * We + (rep ? C : c)) * 3;
                const double l = 0.2126 * (double)p[0] + 0.7152 * (double)p[1] + 0.0722 * (double)p[2];
                if (isfinite(l)) m = fmax(m, l);
            }
        }
    }
    return m;
}

// one CTA per row: the row's weight (fp64) and its column CDF.  Thread t owns a contiguous run of cells; the runs'
// sums are combined in thread order, so the result does not depend on scheduling.
__global__ void __launch_bounds__(IS_BUILD_THREADS) env_sampler_rows_kernel(const float* __restrict__ env, int He, int We,
                                                                            float* table) {
    __shared__ double s_part[IS_BUILD_THREADS + 1];
    const int j = blockIdx.x, C = We - 1;
    const int run = (C + IS_BUILD_THREADS - 1) / IS_BUILD_THREADS;
    const int i0 = min((int)threadIdx.x * run, C), i1 = min(i0 + run, C);
    const double omega = cell_solid_angle(j, He, We);
    double s = 0.0;
    for (int i = i0; i < i1; ++i) s += cell_max_lum(env, He, We, j, i) * omega;
    s_part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {                                  // exclusive prefix of the runs, in order
        double acc = 0.0;
        for (int t = 0; t < IS_BUILD_THREADS; ++t) { const double v = s_part[t]; s_part[t] = acc; acc += v; }
        s_part[IS_BUILD_THREADS] = acc;
        reinterpret_cast<double*>(table + 4)[j] = acc;
        if (j == 0) { table[0] = __int_as_float(He); table[1] = __int_as_float(We); table[2] = table[3] = 0.f; }
    }
    __syncthreads();
    const double total = s_part[IS_BUILD_THREADS];
    float* cc = table + 4 + 2 * (size_t)He + 3 * ((size_t)He + 1) + (size_t)j * We;
    double acc = s_part[threadIdx.x];
    for (int i = i0; i < i1; ++i) {
        cc[i] = total > 0.0 ? (float)(acc / total) : (float)((double)i / C);
        acc += cell_max_lum(env, He, We, j, i) * omega;
    }
    if (threadIdx.x == 0) { cc[0] = 0.f; cc[C] = 1.f; }
}

// the row CDF (the rows' weights in row order; solid angles when every weight is 0) and 1 -+ cos of the band edges
// (2 sin^2 and 2 cos^2 of the half angle: no cancellation)
__global__ void __launch_bounds__(IS_BUILD_THREADS) env_sampler_marginal_kernel(int He, float* table) {
    const double* w = reinterpret_cast<const double*>(table + 4);
    float* rc = table + 4 + 2 * (size_t)He;
    float *vs = rc + He + 1, *cv = vs + He + 1;
    for (int j = threadIdx.x + 1; j < He; j += IS_BUILD_THREADS) {
        const double h = 0.5 * (j - 0.5) * (M_PI / (He - 1)), s = sin(h), c = cos(h);
        vs[j] = (float)(2.0 * s * s); cv[j] = (float)(2.0 * c * c);
    }
    if (threadIdx.x != 0) return;
    vs[0] = 0.f; vs[He] = 2.f; cv[0] = 2.f; cv[He] = 0.f;
    double total = 0.0;
    for (int j = 0; j < He; ++j) total += w[j];
    const bool uniform = !(total > 0.0);
    if (uniform) {
        total = 0.0;
        for (int j = 0; j < He; ++j) total += cos(band_lo(j, He)) - cos(band_hi(j, He));
    }
    double acc = 0.0;
    for (int j = 0; j < He; ++j) {
        rc[j] = (float)(acc / total);
        acc += uniform ? cos(band_lo(j, He)) - cos(band_hi(j, He)) : w[j];
    }
    rc[0] = 0.f; rc[He] = 1.f;
}

// cell pdf = P(row) P(column | row) / solid angle, from the rounded CDFs the sampler inverts
__global__ void env_sampler_pdf_kernel(int He, int We, float* table) {
    const int C = We - 1;
    const float* rc = table + 4 + 2 * (size_t)He;
    const float* cc = rc + 3 * ((size_t)He + 1);
    float* pdf = const_cast<float*>(cc) + (size_t)He * We;
    for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < (size_t)He * C; c += (size_t)gridDim.x * blockDim.x) {
        const int j = (int)(c / C), i = (int)(c - (size_t)j * C);
        const double pr = (double)rc[j + 1] - (double)rc[j];
        const double pc = (double)cc[(size_t)j * We + i + 1] - (double)cc[(size_t)j * We + i];
        pdf[c] = (float)(pr * pc / cell_solid_angle(j, He, We));
    }
}

// one thread per (row, sample)
__global__ void __launch_bounds__(256) importance_dirs_kernel(int P, ImportanceSampler s, const float* __restrict__ table,
                                                              const float* __restrict__ normals, const float* __restrict__ viewdirs,
                                                              const float* __restrict__ roughness, float* __restrict__ dirs,
                                                              float* __restrict__ areas) {
    s.t = EnvTable(table);
    const long long total = (long long)P * s.N;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < total; r += (long long)gridDim.x * blockDim.x) {
        const int g = (int)(r / s.N), i = (int)(r - (long long)g * s.N);
        const float3 nh = unit_normal(normals[3 * (size_t)g], normals[3 * (size_t)g + 1], normals[3 * (size_t)g + 2]);
        GgxFrame f{};
        if (s.n_ggx > 0)
            f = ggx_frame(nh, viewdirs[3 * (size_t)g], viewdirs[3 * (size_t)g + 1], viewdirs[3 * (size_t)g + 2], roughness[g]);
        float area;
        const float3 d = importance_sample(s, (uint32_t)g, i, nh, f, area);
        dirs[3 * r] = d.x; dirs[3 * r + 1] = d.y; dirs[3 * r + 2] = d.z;
        areas[r] = area;
    }
}

}  // namespace r3dg

using namespace r3dg;
extern "C" {

size_t r3dg_env_sampler_floats(int env_h, int env_w) {
    return env_h < 2 || env_w < 2 ? 0 : env_sampler_floats(env_h, env_w);
}

int r3dg_env_sampler_build(const float* env, int env_h, int env_w, float* table, r3dg_stream_t stream_) {
    if (!env || !table || env_h < 2 || env_w < 2) return R3DG_ERR_BAD_ARG;
    if ((long long)env_h * env_w > 0x7fffffffLL / 3) return R3DG_ERR_UNSUPPORTED;
    const cudaStream_t stream = (cudaStream_t)stream_;
    env_sampler_rows_kernel<<<env_h, IS_BUILD_THREADS, 0, stream>>>(env, env_h, env_w, table);
    R3DG_CUDA_TRY(cudaGetLastError());
    env_sampler_marginal_kernel<<<1, IS_BUILD_THREADS, 0, stream>>>(env_h, table);
    R3DG_CUDA_TRY(cudaGetLastError());
    const long long cells = (long long)env_h * (env_w - 1);
    const int blocks = (int)std::min<long long>((cells + 255) / 256, (long long)num_sms() * 8);
    env_sampler_pdf_kernel<<<blocks, 256, 0, stream>>>(env_h, env_w, table);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int r3dg_sample_importance_dirs(int P, int N, const float* normals, const float* viewdirs, const float* roughness,
                                const float* table, const float* env_transform, int n_env, int n_ggx,
                                unsigned long long seed, float* dirs, float* areas, r3dg_stream_t stream_) {
    if (P < 0 || N < 1 || n_env < 0 || n_ggx < 0 || (long long)N - n_env - n_ggx < 1 || seed > 0xffffffffull)
        return R3DG_ERR_BAD_ARG;
    if (n_ggx > 0 && (!viewdirs || !roughness)) return R3DG_ERR_BAD_ARG;
    if (P == 0) return 0;
    if (!normals || !table || !dirs || !areas) return R3DG_ERR_BAD_ARG;
    ImportanceSampler s{};
    s.T = env_transform; s.N = N; s.n_env = n_env; s.n_ggx = n_ggx; s.seed = (uint32_t)seed;
    const long long total = (long long)P * N;
    const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)num_sms() * 16);
    importance_dirs_kernel<<<blocks, 256, 0, (cudaStream_t)stream_>>>(P, s, table, normals, viewdirs, roughness, dirs, areas);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // extern "C"
