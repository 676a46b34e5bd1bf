// Multi-GPU exchange step (SURVEY.md §8e): rebuild the view-averaged SH gradient from the
// all-gathered per-view rank-1 factors instead of all-reducing the dense [P,M,3] tensor.
//
// For one view the reference's SH backward (backward.cu:20-139) gives
//     dL_dsh[g,k,:] = basis_k(normalize(mean_g - campos)) * f[g,:],    f = clamp-gated dL_dRGB
// so 192 B of every Gaussian's 248 B gradient row are an outer product of 16 numbers every rank can
// recompute (means3D is replicated, the step's camera centres are known to all ranks) with 3
// numbers only the rendering rank has.  Exchanging f (12 B per Gaussian and view, all-gather)
// and summing the outer products locally replaces 2*(N-1)/N * 192 B of all-reduce traffic per
// Gaussian and GPU by (N-1) * 12 B, and the projection backward no longer writes the dense tensor.
//
// Design notes: HBM-bound (reads 12 B + N*12 B, writes 192 B per Gaussian); one thread per
// Gaussian accumulates its 3*M values in a transposed shared slab column (conflict-free), the CTA
// writes the [128][3M] slab back with coalesced 16-byte stores — the same slab scheme as
// projection_bwd.cu.  The basis is evaluated with the expressions of projection_bwd.cu so a
// one-view "exchange" reproduces that kernel's dL_dsh.
#include "common.cuh"
#include "kernels.h"

namespace r3dg {

#define SHX_THREADS 128
#define SHX_LD (SHX_THREADS + 1)
#define SHX_MAX_VIEWS 64

struct ShxParams {
    int P, D, M, num_views;
    const float *means3D, *campos;
    const float* factors[SHX_MAX_VIEWS];       // view v's [P,3] factor rows: local memory (all-gathered) or PEER memory
    float scale;
    float* dL_dsh;
    // optional second job of the same launch: in-place mean over the ranks of a flat fp32 section that exists at the
    // same offset in every rank's symmetric buffer (the dense per-Gaussian gradients)
    int rank, sh_blocks;
    long long n_dense4;                         // float4 elements of the section (0: no dense job)
    float* dense_peers[SHX_MAX_VIEWS];          // the section on every rank (peer pointers; [rank] is local)
    float* dense_mc;                            // multicast (NVLS) address of the section, or nullptr
};

__device__ __forceinline__ void shx_basis(int D, float x, float y, float z, float* w) {
#pragma unroll
    for (int k = 0; k < 16; ++k) w[k] = 0.f;
    const float C1 = 0.4886025119029199f;
    w[0] = 0.28209479177387814f;
    if (D > 0) {
        w[1] = -C1 * y; w[2] = C1 * z; w[3] = -C1 * x;
        if (D > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            w[4] = 1.0925484305920792f * xy; w[5] = -1.0925484305920792f * yz; w[6] = 0.31539156525252005f * (2.f * zz - xx - yy);
            w[7] = -1.0925484305920792f * xz; w[8] = 0.5462742152960396f * (xx - yy);
            if (D > 2) {
                w[9] = -0.5900435899266435f * y * (3.f * xx - yy); w[10] = 2.890611442640554f * xy * z;
                w[11] = -0.4570457994644658f * y * (4.f * zz - xx - yy);
                w[12] = 0.3731763325901154f * z * (2.f * zz - 3.f * xx - 3.f * yy);
                w[13] = -0.4570457994644658f * x * (4.f * zz - xx - yy);
                w[14] = 1.445305721320277f * z * (xx - yy); w[15] = -0.5900435899266435f * x * (xx - 3.f * yy);
            }
        }
    }
}

// ---- NVLink all-reduce (mean) of a flat section, fused into the exchange launch -------------------------------------
// Rank r owns the r-th slice.  With a multicast mapping (NVSwitch NVLS) one `multimem.ld_reduce` pulls the 16 bytes
// from every GPU and adds them INSIDE the switch, one `multimem.st` writes the mean back into every GPU's copy: each
// link carries every byte once per direction.  Without multicast the slice is summed with peer loads (in rank order)
// and broadcast with peer stores.  The caller brackets the launch with cross-rank barriers.
__device__ __forceinline__ void dense_mean_slice(const ShxParams& p, int block, int nblocks) {
    const long long per = (p.n_dense4 + p.num_views - 1) / p.num_views;
    const long long lo = min((long long)p.rank * per, p.n_dense4), hi = min(lo + per, p.n_dense4);
    const float s = p.scale;
    for (long long i = lo + (long long)block * SHX_THREADS + threadIdx.x; i < hi; i += (long long)nblocks * SHX_THREADS) {
        float4 v;
        if (p.dense_mc) {
            float4* a = reinterpret_cast<float4*>(p.dense_mc) + i;
            asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                         : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(a) : "memory");
            v.x *= s; v.y *= s; v.z *= s; v.w *= s;
            asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
        } else {
            v = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < p.num_views; ++r) {
                const float4 t = reinterpret_cast<const float4*>(p.dense_peers[r])[i];
                v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
            }
            v.x *= s; v.y *= s; v.z *= s; v.w *= s;
            for (int r = 0; r < p.num_views; ++r) reinterpret_cast<float4*>(p.dense_peers[r])[i] = v;
        }
    }
    __threadfence_system();
}

__global__ void __launch_bounds__(SHX_THREADS) sh_from_factors_kernel(const ShxParams p) {
    extern __shared__ float sOut[];                       // [3M][SHX_LD]
    __shared__ float sCam[3 * SHX_MAX_VIEWS];
    // The dense-mean job rides in the same launch, its CTAs INTERLEAVED with the rebuild CTAs (every `period`-th block)
    // so that the NVLink-bound reduction and the HBM-write-bound rebuild run side by side instead of one after the other.
    const int dense_blocks = (int)gridDim.x - p.sh_blocks;
    int sh_block = (int)blockIdx.x;
    if (dense_blocks > 0) {
        const int period = max(1, (int)gridDim.x / dense_blocks);
        const int b = (int)blockIdx.x;
        const int q = b / period;                              // dense blocks at b = 0, period, 2 period, ... while q < dense_blocks
        if (b % period == 0 && q < dense_blocks) { dense_mean_slice(p, q, dense_blocks); return; }
        sh_block = b - min(dense_blocks, q + 1);               // dense blocks seen so far: indices 0..q (or all of them)
    }
    for (int i = threadIdx.x; i < 3 * p.num_views; i += SHX_THREADS) sCam[i] = p.campos[i];
    __syncthreads();
    const int block_base = sh_block * SHX_THREADS;
    const int idx = block_base + threadIdx.x;
    const int rowf = 3 * p.M;
    const int nvalid = min(SHX_THREADS, p.P - block_base);
    if (idx < p.P) {
        const float mx = p.means3D[3 * (size_t)idx], my = p.means3D[3 * (size_t)idx + 1], mz = p.means3D[3 * (size_t)idx + 2];
        float acc[48];
#pragma unroll
        for (int q = 0; q < 48; ++q) acc[q] = 0.f;
        // factors of 8 views at a time: all (peer) loads are issued before any is used, so their NVLink latencies overlap
        for (int v0 = 0; v0 < p.num_views; v0 += 8) {
            float f[8][3];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                f[u][0] = f[u][1] = f[u][2] = 0.f;
                if (v0 + u < p.num_views) {
                    const float* src = p.factors[v0 + u] + (size_t)idx * 3;       // peer memory in the P2P exchange: coalesced 12 B/thread NVLink reads
                    f[u][0] = src[0]; f[u][1] = src[1]; f[u][2] = src[2];
                }
            }
#pragma unroll 1
            for (int u = 0; u < 8; ++u) {
                const int v = v0 + u;
                float f0 = f[0][0], f1 = f[0][1], f2 = f[0][2];
#pragma unroll
                for (int t = 1; t < 8; ++t)
                    if (u == t) { f0 = f[t][0]; f1 = f[t][1]; f2 = f[t][2]; }       // register select (no local-memory indexing)
                if (v >= p.num_views || (f0 == 0.f && f1 == 0.f && f2 == 0.f)) continue;   // culled in this view (or fully clamped): exact zeros
                const float dox = mx - sCam[3 * v], doy = my - sCam[3 * v + 1], doz = mz - sCam[3 * v + 2];
                const float len = sqrtf(dox * dox + doy * doy + doz * doz);
                float w[16];
                shx_basis(p.D, dox / len, doy / len, doz / len, w);
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    acc[3 * k] += w[k] * f0; acc[3 * k + 1] += w[k] * f1; acc[3 * k + 2] += w[k] * f2;
                }
            }
        }
        float* col = sOut + threadIdx.x;
#pragma unroll
        for (int k = 0; k < 16; ++k)
            if (k < p.M) {
                col[(3 * k) * SHX_LD] = acc[3 * k] * p.scale;
                col[(3 * k + 1) * SHX_LD] = acc[3 * k + 1] * p.scale;
                col[(3 * k + 2) * SHX_LD] = acc[3 * k + 2] * p.scale;
            }
    }
    __syncthreads();
    const int total = nvalid * rowf;
    float* dst = p.dL_dsh + (size_t)block_base * rowf;
    if ((rowf & 3) == 0) {
        float4* dst4 = reinterpret_cast<float4*>(dst);
        for (int i4 = threadIdx.x; i4 < total / 4; i4 += SHX_THREADS) {
            const int i = 4 * i4, t = i / rowf, k = i - t * rowf;
            dst4[i4] = make_float4(sOut[(k + 0) * SHX_LD + t], sOut[(k + 1) * SHX_LD + t], sOut[(k + 2) * SHX_LD + t], sOut[(k + 3) * SHX_LD + t]);
        }
    } else {
        for (int i = threadIdx.x; i < total; i += SHX_THREADS) {
            const int t = i / rowf, k = i - t * rowf;
            dst[i] = sOut[k * SHX_LD + t];
        }
    }
}

}  // namespace r3dg

using namespace r3dg;
extern "C" {

unsigned long long r3dg_shx_launches = 0;      // folded into r3dg_launch_count (api.cu)

static int launch_shx(ShxParams& p, int dense_blocks, cudaStream_t stream) {
    const size_t smem = (size_t)3 * p.M * SHX_LD * sizeof(float);
    p.sh_blocks = (p.P + SHX_THREADS - 1) / SHX_THREADS;
    sh_from_factors_kernel<<<p.sh_blocks + dense_blocks, SHX_THREADS, smem, stream>>>(p);
    R3DG_CUDA_TRY(cudaGetLastError());
    ++r3dg_shx_launches;
    return 0;
}

int r3dg_sh_grad_from_factors(int P, int D, int M, int num_views, const float* means3D, const float* campos,
                              const float* factors, float scale, float* dL_dsh, r3dg_stream_t stream) {
    if (P < 0 || D < 0 || D > 3 || M < 1 || M > 16 || (D + 1) * (D + 1) > M || num_views < 1) return R3DG_ERR_BAD_ARG;
    if (num_views > SHX_MAX_VIEWS) return R3DG_ERR_UNSUPPORTED;
    if (P == 0) return 0;
    if (!means3D || !campos || !factors || !dL_dsh) return R3DG_ERR_BAD_ARG;
    ShxParams p = {};
    p.P = P; p.D = D; p.M = M; p.num_views = num_views;
    p.means3D = means3D; p.campos = campos; p.scale = scale; p.dL_dsh = dL_dsh;
    for (int v = 0; v < num_views; ++v) p.factors[v] = factors + (size_t)v * P * 3;
    return launch_shx(p, 0, (cudaStream_t)stream);
}

int r3dg_exchange_p2p(const r3dg_exchange_args* a, r3dg_stream_t stream) {
    if (!a || a->P < 0 || a->D < 0 || a->D > 3 || a->M < 1 || a->M > 16 || (a->D + 1) * (a->D + 1) > a->M) return R3DG_ERR_BAD_ARG;
    if (a->world < 1 || a->world > SHX_MAX_VIEWS || a->rank < 0 || a->rank >= a->world) return R3DG_ERR_BAD_ARG;
    if (a->n_dense < 0 || (a->n_dense & 3)) return R3DG_ERR_BAD_ARG;
    if (a->P == 0 && a->n_dense == 0) return 0;
    if (a->P > 0 && (!a->means3D || !a->campos || !a->dL_dsh)) return R3DG_ERR_BAD_ARG;
    ShxParams p = {};
    p.P = a->P; p.D = a->D; p.M = a->M; p.num_views = a->world; p.rank = a->rank;
    p.means3D = a->means3D; p.campos = a->campos; p.scale = 1.0f / (float)a->world; p.dL_dsh = a->dL_dsh;
    for (int v = 0; v < a->world; ++v) {
        p.factors[v] = a->factors[v]; p.dense_peers[v] = a->dense[v];
        if (a->P > 0 && !a->factors[v]) return R3DG_ERR_BAD_ARG;
        if (a->n_dense > 0 && !a->dense[v]) return R3DG_ERR_BAD_ARG;
    }
    p.n_dense4 = a->n_dense / 4; p.dense_mc = a->dense_multicast;
    // enough CTAs to keep the NVLink pipes full; the SH rebuild blocks run beside them
    const int dense_blocks = a->n_dense > 0 ? 1184 : 0;
    return launch_shx(p, dense_blocks, (cudaStream_t)stream);
}

}  // extern "C"
