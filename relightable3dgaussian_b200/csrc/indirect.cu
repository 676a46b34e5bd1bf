// Ray-traced indirect light: the radiance bake (front-to-back compositing of the Gaussians each incident ray of the
// visibility bake meets) and the per-Gaussian least-squares fit of its result into incident-light SH
// (the reference's `incidents`, scene/gaussian_model.py:394,450).
//
// Design notes (DESIGN.md §4.25)
//  * rays, hit set and tree are the visibility bake's (bvh.cu): same packed tree, same directions, same slab test
//    deciding which children are visited, same per-Gaussian hit arithmetic.  Only the ORDER is new: radiance is
//    composited in ascending (t, Gaussian index).
//  * k-buffer rounds: each round walks the tree once and keeps, in registers, the RAD_K smallest hit keys above the
//    last composited key; it then composites them in order.  A round that ends with a free buffer entry has seen
//    every remaining hit.  Nothing depends on the traversal order, so the bake is bitwise reproducible.
//  * a hit's t need not lie inside its own 3-sigma box (a ray that clips a box corner peaks outside it), so box
//    intervals do not bound the keys below a subtree: the only cull is the visibility trace's own "box hit" test.
//  * the fit: one warp per Gaussian, Gram matrix and right-hand side in fp64 summed in sample order, one lane
//    per matrix entry, then a Cholesky solve — deterministic.
#include "bvh.cuh"
#include "kernels.h"
#include "sh.cuh"

namespace r3dg {

#define RAD_THREADS 128
#define RAD_K 16                // k-buffer entries per round
#define RAD_T_MIN 1e-4f         // a ray stops once its transmittance falls below this

// Ray r = (leaf slot r / N, sample r % N): rays in Morton order, results at the Gaussian's own row g * N + i.
__global__ void __launch_bounds__(RAD_THREADS) bvh_radiance_kernel(int P, int N, const float4* __restrict__ packets,
                                                                   const int32_t* __restrict__ nodes,
                                                                   const float* __restrict__ shs, int M, int deg,
                                                                   float o_offset, float* __restrict__ radiance,
                                                                   float* __restrict__ transmittance,
                                                                   int32_t* __restrict__ num_hits) {
    __shared__ int sStack[TRACE_STACK_SH][RAD_THREADS];
    extern __shared__ float3 sSample[];
    for (int i = threadIdx.x; i < N; i += RAD_THREADS) sSample[i] = fib_sample(i, N);
    __syncthreads();
    const long long ray = (long long)blockIdx.x * RAD_THREADS + threadIdx.x;
    if (ray >= (long long)P * N) return;
    const int NI = P - 1;
    const int slot = (int)(ray / N), i = (int)(ray - (long long)slot * N);
    const LeafRecord self = load_leaf(packets + (size_t)(NI + slot) * 4);
    const float3 d = rotate_from_z(self.nx, self.ny, self.nz, sSample[i]);
    const float dx = d.x, dy = d.y, dz = d.z;
    float o[3] = {self.mx, self.my, self.mz};
    if (o_offset != 0.0f) { o[0] = add_(o[0], mul_(dx, o_offset)); o[1] = add_(o[1], mul_(dy, o_offset)); o[2] = add_(o[2], mul_(dz, o_offset)); }
    const float ox = o[0], oy = o[1], oz = o[2];
    const float ix = div_(1.0f, dx), iy = div_(1.0f, dy), iz = div_(1.0f, dz);
    SplitStack<RAD_THREADS> st;
    st.sh = sStack; st.tid = threadIdx.x;
    const unsigned long long EMPTY = ~0ull;
    unsigned long long last = 0;           // key of the last composited hit; every key is > 0 (t >= 0.01)
    float L0 = 0.f, L1 = 0.f, L2 = 0.f, T = 1.0f;
    int hits = 0;
    bool more = true;
    while (more) {
        // ---- one round: the RAD_K smallest keys (t bits : Gaussian index) above `last`, sorted ascending ----
        unsigned long long key[RAD_K];
        int kslot[RAD_K];
#pragma unroll
        for (int j = 0; j < RAD_K; ++j) { key[j] = EMPTY; kslot[j] = 0; }
        st.sp = 0;
        st.push(NI == 0 ? -1 : 0);        // root (a lone leaf when P == 1)
        while (st.sp > 0) {
            const int node = st.pop();
            if (node >= 0) {
                const float4* p = packets + (size_t)node * 4;
                const float4 p0 = p[0], p1 = p[1], p2 = p[2], p3 = p[3];
                if (ray_box_tmax(p0.z, p0.w, p1.x, p1.y, p1.z, p1.w, ox, oy, oz, ix, iy, iz) > 0) st.push(__float_as_int(p0.x));
                if (ray_box_tmax(p2.x, p2.y, p2.z, p2.w, p3.x, p3.y, ox, oy, oz, ix, iy, iz) > 0) st.push(__float_as_int(p0.y));
            } else {
                const int s = -node - 1;
                const LeafRecord q = load_leaf(packets + (size_t)(NI + s) * 4);
                float t, power;
                if (!gaussian_hit(q, ox, oy, oz, dx, dy, dz, t, power)) continue;
                const unsigned long long k = ((unsigned long long)__float_as_uint(t) << 32) |
                                             (unsigned)nodes[(size_t)(NI + s) * 5 + 3];
                if (k <= last || k >= key[RAD_K - 1]) continue;
                // insertion into the sorted register buffer (keys are unique: one per Gaussian)
#pragma unroll
                for (int j = RAD_K - 1; j > 0; --j) {
                    if (key[j - 1] > k) { key[j] = key[j - 1]; kslot[j] = kslot[j - 1]; }
                    else if (key[j] > k) { key[j] = k; kslot[j] = s; }
                }
                if (key[0] > k) { key[0] = k; kslot[0] = s; }
            }
        }
        more = key[RAD_K - 1] != EMPTY;   // a full buffer may have left hits for the next round
        // ---- composite the round front to back: alpha and colour recomputed from the leaf record and the payload ----
        while (key[0] != EMPTY) {
            const LeafRecord q = load_leaf(packets + (size_t)(NI + kslot[0]) * 4);
            float t, power;
            gaussian_hit(q, ox, oy, oz, dx, dy, dz, t, power);
            const float alpha = q.op * __expf(power);
            float rgb[3];
            unsigned clamped;
            sh_to_rgb(deg, q.mx, q.my, q.mz, o, shs + (size_t)(unsigned)key[0] * M * 3, 1, rgb, clamped);
            const float w = T * alpha;
            L0 += w * rgb[0]; L1 += w * rgb[1]; L2 += w * rgb[2];
            T *= 1 - alpha;
            ++hits;
            last = key[0];
            if (T < RAD_T_MIN) { more = false; break; }
#pragma unroll
            for (int j = 0; j < RAD_K - 1; ++j) { key[j] = key[j + 1]; kslot[j] = kslot[j + 1]; }
            key[RAD_K - 1] = EMPTY;
        }
    }
    const long long out = (long long)nodes[(size_t)(NI + slot) * 5 + 3] * N + i;
    radiance[3 * out] = L0; radiance[3 * out + 1] = L1; radiance[3 * out + 2] = L2;
    transmittance[out] = T;
    if (num_hits) num_hits[out] = hits;
}

// ---- incident-SH fit: min_c (1/N) sum_i |Y(w_i)^T c - L_i|^2 + ridge |c|^2, one warp per Gaussian ---------------
#define FIT_THREADS 128
#define FIT_WARPS (FIT_THREADS / 32)
struct FitWarp {
    float w[32][17];            // basis of the chunk's 32 samples (padded row)
    float L[32][3];             // their radiance
    double G[16][17];           // Gram matrix (Cholesky factor in place), padded row
    double b[16][3];            // right-hand side, then the solution
};

__global__ void __launch_bounds__(FIT_THREADS) fit_incident_sh_kernel(int P, int N, const float* __restrict__ radiance,
                                                                      const float* __restrict__ normals, int deg,
                                                                      double ridge, float* __restrict__ out) {
    __shared__ FitWarp sW[FIT_WARPS];
    extern __shared__ float3 sSample[];
    for (int i = threadIdx.x; i < N; i += FIT_THREADS) sSample[i] = fib_sample(i, N);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = blockIdx.x * FIT_WARPS + warp;
    if (g >= P) return;
    FitWarp& s = sW[warp];
    const int n = (deg + 1) * (deg + 1), ntri = n * (n + 1) / 2, nent = ntri + 3 * n;
    // lane's entries e = lane + 32 q: Gram (a, b) with a <= b for e < ntri, else rhs (k, channel)
    int ea[6], eb[6];
    double acc[6];
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        const int e = lane + 32 * q;
        acc[q] = 0.0;
        if (e < ntri) {
            int a = 0, r = e;
            while (r >= n - a) { r -= n - a; ++a; }
            ea[q] = a; eb[q] = a + r;
        } else {
            ea[q] = (e - ntri) / 3; eb[q] = -1 - (e - ntri) % 3;       // < 0: channel of the rhs
        }
    }
    const float nx = normals[3 * (size_t)g], ny = normals[3 * (size_t)g + 1], nz = normals[3 * (size_t)g + 2];
    for (int base = 0; base < N; base += 32) {
        const int i = base + lane;
        if (i < N) {
            const float3 dir = rotate_from_z(nx, ny, nz, sSample[i]);
            float w[16];
            sh_basis(deg, dir.x, dir.y, dir.z, w);
#pragma unroll
            for (int k = 0; k < 16; ++k) if (k < n) s.w[lane][k] = w[k];
            const float* Li = radiance + ((size_t)g * N + i) * 3;
            s.L[lane][0] = Li[0]; s.L[lane][1] = Li[1]; s.L[lane][2] = Li[2];
        }
        __syncwarp();
        const int cnt = min(32, N - base);
#pragma unroll
        for (int q = 0; q < 6; ++q) {
            if (lane + 32 * q >= nent) continue;
            const int a = ea[q], bb = eb[q];
            double v = acc[q];
            for (int j = 0; j < cnt; ++j)
                v = fma((double)s.w[j][a], bb >= 0 ? (double)s.w[j][bb] : (double)s.L[j][-1 - bb], v);
            acc[q] = v;
        }
        __syncwarp();
    }
    const double inv_n = 1.0 / (double)N;
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        if (lane + 32 * q >= nent) continue;
        const int a = ea[q], bb = eb[q];
        if (bb >= 0) {
            const double v = acc[q] * inv_n + (a == bb ? ridge : 0.0);
            s.G[a][bb] = v; s.G[bb][a] = v;
        } else {
            s.b[a][-1 - bb] = acc[q] * inv_n;
        }
    }
    __syncwarp();
    // Cholesky G = L L^T in place (lower triangle), lane r owns row r
    for (int k = 0; k < n; ++k) {
        const double dkk = sqrt(s.G[k][k]);
        __syncwarp();
        if (lane == k) s.G[k][k] = dkk;
        if (lane > k && lane < n) s.G[lane][k] /= dkk;
        __syncwarp();
        if (lane > k && lane < n)
            for (int c = k + 1; c <= lane; ++c) s.G[lane][c] -= s.G[lane][k] * s.G[c][k];
        __syncwarp();
    }
    // L y = b, then L^T x = y: lane c < 3 solves channel c
    if (lane < 3) {
        for (int r = 0; r < n; ++r) {
            double v = s.b[r][lane];
            for (int c = 0; c < r; ++c) v -= s.G[r][c] * s.b[c][lane];
            s.b[r][lane] = v / s.G[r][r];
        }
        for (int r = n - 1; r >= 0; --r) {
            double v = s.b[r][lane];
            for (int c = r + 1; c < n; ++c) v -= s.G[c][r] * s.b[c][lane];
            s.b[r][lane] = v / s.G[r][r];
        }
    }
    __syncwarp();
    for (int e = lane; e < 3 * n; e += 32) out[(size_t)g * 3 * n + e] = (float)s.b[e / 3][e % 3];
}

// ---- host launchers -----------------------------------------------------------------------
size_t bvh_radiance_tmp_bytes(int P) { return bvh_packets_bytes(P); }

int launch_bvh_radiance(int P, int N, const int32_t* nodes, const float* aabbs, const float* means3D, const float* covs3D,
                        const float* opacities, const float* normals, const float* shs, int M, int sh_degree,
                        float o_offset, float* radiance, float* transmittance, int32_t* num_hits, void* tmp,
                        size_t tmp_bytes, cudaStream_t stream) {
    if (P < 0 || N < 0 || sh_degree < 0 || sh_degree > 3 || M < (sh_degree + 1) * (sh_degree + 1)) return R3DG_ERR_BAD_ARG;
    if ((size_t)N * sizeof(float3) > BAKE_SAMPLE_SMEM) return R3DG_ERR_UNSUPPORTED;
    if (P == 0 || N == 0) return 0;
    if (tmp_bytes < bvh_radiance_tmp_bytes(P)) return R3DG_ERR_BAD_ARG;
    float4* packets = (float4*)((char*)tmp + 256);
    const int rc = launch_bvh_pack(P, nodes, aabbs, means3D, covs3D, opacities, normals, packets, stream);
    if (rc != 0) return rc;
    const long long num_rays = (long long)P * N;
    bvh_radiance_kernel<<<(unsigned)((num_rays + RAD_THREADS - 1) / RAD_THREADS), RAD_THREADS, (size_t)N * sizeof(float3), stream>>>(
        P, N, packets, nodes, shs, M, sh_degree, o_offset, radiance, transmittance, num_hits);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_fit_incident_sh(int P, int N, const float* radiance, const float* normals, int degree, float ridge, float* out,
                           cudaStream_t stream) {
    if (P < 0 || N < 0 || degree < 0 || degree > 3 || !(ridge > 0.0f) || !(ridge < 3.0e38f)) return R3DG_ERR_BAD_ARG;
    if ((size_t)N * sizeof(float3) > BAKE_SAMPLE_SMEM) return R3DG_ERR_UNSUPPORTED;
    if (P == 0) return 0;
    if (N == 0) return R3DG_ERR_BAD_ARG;                    // no samples: nothing to fit
    const size_t smem = (size_t)N * sizeof(float3);
    R3DG_CUDA_TRY(cudaFuncSetAttribute(fit_incident_sh_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BAKE_SAMPLE_SMEM));
    fit_incident_sh_kernel<<<(P + FIT_WARPS - 1) / FIT_WARPS, FIT_THREADS, smem, stream>>>(P, N, radiance, normals, degree,
                                                                                           (double)ridge, out);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
