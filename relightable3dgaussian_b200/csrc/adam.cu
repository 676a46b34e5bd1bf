// SURVEY.md §8(f) next #3: the optimiser step either side of the hot path.  The reference updates
// its 7 (stage 1) to 13 (stage 2) per-Gaussian parameter groups with
// `torch.optim.Adam(l, lr=0.0, eps=1e-15)` (scene/gaussian_model.py:465-497), i.e. per group the
// chain exp_avg.mul_().add_() / exp_avg_sq.mul_().addcmul_() / sqrt / div / add_ / addcdiv_ of
// torch 1.12.1's `_single_tensor_adam` (torch/optim/adam.py; torch is a dependency, not part of
// /root/reference) — ~8 elementwise kernels and ~60 B of HBM traffic per element and group.
// Here ONE launch updates every group: 28 B per element (read p, g, m, v; write p, m, v), the
// HBM floor for Adam with fp32 state.
//
// Design notes
//  * the descriptor table (<= 16 tensors) travels in the kernel parameter space; blocks are dealt
//    over the concatenation of all tensors in units of 4096 elements, a block finds its tensor
//    with a <= 16-step scan of the block prefix;
//  * 128-bit loads/stores, 4 independent float4 chains per thread (16 elements) to cover HBM
//    latency; tensors whose four pointers are not 16-byte aligned take the scalar path;
//  * the scalar factors (step size lr / (1 - beta1^t), 1 / sqrt(1 - beta2^t)) are computed on the
//    host in double precision exactly like torch's Python code and passed as floats.
//  * selective step (a row mask per tensor): a second instantiation of the same kernel.  Each float4
//    (each element on the scalar path) works out the 1-4 rows it covers and reads their mask bytes;
//    with none set it loads and stores nothing, gradient included.  Otherwise only the set rows'
//    elements are updated and the others are written back with the bits that were loaded.  No scan
//    or compaction: a compacted row list would need a count read-back or a second launch, while
//    the gated sweep reads one mask byte per row within the one launch.
#include <climits>
#include <cmath>
#include "common.cuh"
#include "kernels.h"

namespace r3dg {

#define ADAM_THREADS 256
#define ADAM_ILP 4
#define ADAM_BLOCK_ELEMS (ADAM_THREADS * 4 * ADAM_ILP)      // 4096 elements per block
#define ADAM_MAX_TENSORS 16

struct AdamTensor {
    float* p;
    const float* g;
    float* m;
    float* v;
    long long n;
    float step_size;         // lr / bias_correction1
    float inv_bc2_sqrt;      // 1 / sqrt(bias_correction2)
    float beta1, beta2, one_minus_beta1, one_minus_beta2, eps;
    int vec;                 // all four pointers 16-byte aligned
};

struct AdamTable {
    AdamTensor t[ADAM_MAX_TENSORS];
    long long block_end[ADAM_MAX_TENSORS];     // exclusive prefix of blocks per tensor
    int num;
};

// Kernel parameters: the dense step passes the table alone; the selective step adds, per tensor, its row mask
// (NULL: the dense body) and elements per row.  A separate struct keeps the dense parameter layout as it was.
template <bool MASKED> struct AdamArgs { AdamTable tab; };
template <> struct AdamArgs<true> {
    AdamTable tab;
    const unsigned char* row_mask[ADAM_MAX_TENSORS];
    long long row_elems[ADAM_MAX_TENSORS];
};

// torch 1.12.1 torch/optim/adam.py:_single_tensor_adam, one element
__device__ __forceinline__ void adam_update(const AdamTensor& t, float& p, float g, float& m, float& v) {
    m = __fadd_rn(__fmul_rn(m, t.beta1), __fmul_rn(g, t.one_minus_beta1));          // exp_avg.mul_(beta1).add_(grad, alpha=1-beta1)
    v = __fadd_rn(__fmul_rn(v, t.beta2), __fmul_rn(__fmul_rn(t.one_minus_beta2, g), g));   // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1-beta2)
    // denom = (exp_avg_sq.sqrt() / sqrt(bc2)).add_(eps);  param.addcdiv_(exp_avg, denom, value=-step_size).
    // The two moments above are the exact per-op IEEE chain (bit-identical to torch's CPU / numpy rounding; torch's own
    // CUDA functors contract mul+add into FMA).  The quotient only scales the UPDATE, so it
    // uses the one-MUFU forms (sqrt.approx, division by reciprocal: <= 2 ulp of the update, ~1e-7 of a step that is itself
    // ~lr): IEEE div / sqrt branch to a slow subroutine whenever an operand is zero or denormal, real gradients are
    // full of exact zeros (Gaussians a view does not see), and one such lane stalls its warp.
    float sq;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(sq) : "f"(v));                      // exact 0 for v == 0, no slow path
    const float denom = __fadd_rn(__fmul_rn(sq, t.inv_bc2_sqrt), t.eps);
    p = __fadd_rn(p, __fmul_rn(-t.step_size, __fdividef(m, denom)));
}

// Selective body for one tensor of rows of `re` elements, row r updated only where mask[r] != 0.  All positions
// inside the block are 32-bit offsets from the block's first element, which lies `rem0` elements into row `row0`.
__device__ __forceinline__ void adam_masked(const AdamTensor& t, const unsigned char* __restrict__ mask, long long re64,
                                            long long base) {
    const unsigned re = (unsigned)re64;                        // r3dg_adam_step refuses row_elems > INT_MAX
    const long long row0 = base / re64;
    const unsigned rem0 = (unsigned)(base - row0 * re64);
    if (t.vec && base + ADAM_BLOCK_ELEMS <= t.n) {
        unsigned on[ADAM_ILP];                                 // bit j: element j of the float4 is in a set row
#pragma unroll
        for (int k = 0; k < ADAM_ILP; ++k) {
            const unsigned s = rem0 + 4u * ((unsigned)k * ADAM_THREADS + threadIdx.x);
            long long row = row0 + s / re;
            unsigned r = s % re;
            unsigned b = __ldg(mask + row) != 0;
#pragma unroll
            for (int j = 1; j < 4; ++j) {
                if (++r == re) { r = 0; b |= (unsigned)(__ldg(mask + ++row) != 0) << j; }
                else b |= (b >> (j - 1) & 1u) << j;
            }
            on[k] = b;
        }
        float4 p4[ADAM_ILP], g4[ADAM_ILP], m4[ADAM_ILP], v4[ADAM_ILP];
#pragma unroll
        for (int k = 0; k < ADAM_ILP; ++k) {
            if (!on[k]) continue;
            const long long i = base + 4 * ((long long)k * ADAM_THREADS + threadIdx.x);
            p4[k] = *reinterpret_cast<const float4*>(t.p + i);
            g4[k] = __ldcs(reinterpret_cast<const float4*>(t.g + i));
            m4[k] = *reinterpret_cast<const float4*>(t.m + i);
            v4[k] = *reinterpret_cast<const float4*>(t.v + i);
        }
#pragma unroll
        for (int k = 0; k < ADAM_ILP; ++k) {
            if (!on[k]) continue;
            if (on[k] & 1u) adam_update(t, p4[k].x, g4[k].x, m4[k].x, v4[k].x);
            if (on[k] & 2u) adam_update(t, p4[k].y, g4[k].y, m4[k].y, v4[k].y);
            if (on[k] & 4u) adam_update(t, p4[k].z, g4[k].z, m4[k].z, v4[k].z);
            if (on[k] & 8u) adam_update(t, p4[k].w, g4[k].w, m4[k].w, v4[k].w);
            const long long i = base + 4 * ((long long)k * ADAM_THREADS + threadIdx.x);
            *reinterpret_cast<float4*>(t.p + i) = p4[k];
            *reinterpret_cast<float4*>(t.m + i) = m4[k];
            *reinterpret_cast<float4*>(t.v + i) = v4[k];
        }
    } else {
        const long long end = base + ADAM_BLOCK_ELEMS < t.n ? base + ADAM_BLOCK_ELEMS : t.n;
        for (long long i = base + threadIdx.x; i < end; i += ADAM_THREADS) {
            if (!__ldg(mask + row0 + (rem0 + (unsigned)(i - base)) / re)) continue;
            float p = t.p[i], m = t.m[i], v = t.v[i];
            adam_update(t, p, t.g[i], m, v);
            t.p[i] = p; t.m[i] = m; t.v[i] = v;
        }
    }
}

template <bool MASKED>
__global__ void __launch_bounds__(ADAM_THREADS) adam_kernel(const __grid_constant__ AdamArgs<MASKED> args) {
    const AdamTable& tab = args.tab;
    int ti = 0;
    while (ti < tab.num - 1 && (long long)blockIdx.x >= tab.block_end[ti]) ++ti;
    const AdamTensor& t = tab.t[ti];
    const long long first_block = ti == 0 ? 0 : tab.block_end[ti - 1];
    const long long base = ((long long)blockIdx.x - first_block) * ADAM_BLOCK_ELEMS;
    if constexpr (MASKED) {
        if (args.row_mask[ti]) {
            adam_masked(t, args.row_mask[ti], args.row_elems[ti], base);
            return;
        }
    }
    if (t.vec && base + ADAM_BLOCK_ELEMS <= t.n) {
        float4 p4[ADAM_ILP], g4[ADAM_ILP], m4[ADAM_ILP], v4[ADAM_ILP];
#pragma unroll
        for (int k = 0; k < ADAM_ILP; ++k) {
            const long long i = base + 4 * ((long long)k * ADAM_THREADS + threadIdx.x);
            p4[k] = *reinterpret_cast<const float4*>(t.p + i);
            g4[k] = __ldcs(reinterpret_cast<const float4*>(t.g + i));       // gradients are dead after the step
            m4[k] = *reinterpret_cast<const float4*>(t.m + i);
            v4[k] = *reinterpret_cast<const float4*>(t.v + i);
        }
#pragma unroll
        for (int k = 0; k < ADAM_ILP; ++k) {
            adam_update(t, p4[k].x, g4[k].x, m4[k].x, v4[k].x);
            adam_update(t, p4[k].y, g4[k].y, m4[k].y, v4[k].y);
            adam_update(t, p4[k].z, g4[k].z, m4[k].z, v4[k].z);
            adam_update(t, p4[k].w, g4[k].w, m4[k].w, v4[k].w);
            const long long i = base + 4 * ((long long)k * ADAM_THREADS + threadIdx.x);
            *reinterpret_cast<float4*>(t.p + i) = p4[k];
            *reinterpret_cast<float4*>(t.m + i) = m4[k];
            *reinterpret_cast<float4*>(t.v + i) = v4[k];
        }
    } else {
        const long long end = base + ADAM_BLOCK_ELEMS < t.n ? base + ADAM_BLOCK_ELEMS : t.n;
        for (long long i = base + threadIdx.x; i < end; i += ADAM_THREADS) {
            float p = t.p[i], m = t.m[i], v = t.v[i];
            adam_update(t, p, t.g[i], m, v);
            t.p[i] = p; t.m[i] = m; t.v[i] = v;
        }
    }
}

int launch_adam(int num, const r3dg_adam_tensor* ts, cudaStream_t stream, int* launches) {
    *launches = 0;
    int i = 0;
    while (i < num) {
        AdamArgs<true> args;                   // .tab alone is the dense launch's parameter block
        AdamTable& tab = args.tab;
        tab.num = 0;
        long long blocks = 0;
        bool masked = false;
        for (; i < num && tab.num < ADAM_MAX_TENSORS; ++i) {
            const r3dg_adam_tensor& s = ts[i];
            if (s.n == 0) continue;
            args.row_mask[tab.num] = s.row_mask;
            args.row_elems[tab.num] = s.row_mask ? s.row_elems : 1;
            masked = masked || s.row_mask;
            // bias corrections exactly as torch's Python code computes them (double precision)
            const double bc1 = 1.0 - pow((double)s.beta1, (double)s.step);
            const double bc2 = 1.0 - pow((double)s.beta2, (double)s.step);
            AdamTensor& t = tab.t[tab.num];
            t.p = s.param; t.g = s.grad; t.m = s.exp_avg; t.v = s.exp_avg_sq; t.n = s.n;
            t.step_size = (float)((double)s.lr / bc1);
            t.inv_bc2_sqrt = (float)(1.0 / sqrt(bc2));
            t.beta1 = (float)s.beta1; t.beta2 = (float)s.beta2;
            t.one_minus_beta1 = (float)(1.0 - s.beta1); t.one_minus_beta2 = (float)(1.0 - s.beta2);
            t.eps = (float)s.eps;
            t.vec = ((((uintptr_t)s.param | (uintptr_t)s.grad | (uintptr_t)s.exp_avg | (uintptr_t)s.exp_avg_sq) & 15) == 0) ? 1 : 0;
            blocks += (s.n + ADAM_BLOCK_ELEMS - 1) / ADAM_BLOCK_ELEMS;
            tab.block_end[tab.num] = blocks;
            ++tab.num;
        }
        if (tab.num == 0) continue;
        if (blocks > 0x7fffffffLL) return R3DG_ERR_UNSUPPORTED;
        for (int k = tab.num; k < ADAM_MAX_TENSORS; ++k) {
            tab.block_end[k] = blocks;
            args.row_mask[k] = nullptr;
            args.row_elems[k] = 1;
        }
        if (masked) adam_kernel<true><<<(unsigned)blocks, ADAM_THREADS, 0, stream>>>(args);
        else adam_kernel<false><<<(unsigned)blocks, ADAM_THREADS, 0, stream>>>(AdamArgs<false>{tab});
        R3DG_CUDA_TRY(cudaGetLastError());
        ++*launches;
    }
    return 0;
}

}  // namespace r3dg

// ---- C ABI --------------------------------------------------------------------------------------
using namespace r3dg;
extern "C" {

unsigned long long r3dg_adam_launches = 0;      // folded into r3dg_launch_count (api.cu)

int r3dg_adam_step(int num_tensors, const r3dg_adam_tensor* tensors, r3dg_stream_t stream) {
    if (num_tensors < 0 || (num_tensors > 0 && !tensors)) return R3DG_ERR_BAD_ARG;
    for (int i = 0; i < num_tensors; ++i) {
        const r3dg_adam_tensor& t = tensors[i];
        if (t.n < 0 || t.step < 1) return R3DG_ERR_BAD_ARG;
        if (t.n > 0 && (!t.param || !t.grad || !t.exp_avg || !t.exp_avg_sq)) return R3DG_ERR_BAD_ARG;
        if (!(t.beta1 >= 0.0 && t.beta1 < 1.0) || !(t.beta2 >= 0.0 && t.beta2 < 1.0) || !(t.eps >= 0.0)) return R3DG_ERR_BAD_ARG;
        if (t.row_mask && (t.row_elems < 1 || t.n % t.row_elems != 0)) return R3DG_ERR_BAD_ARG;
        if (t.row_mask && t.row_elems > INT_MAX) return R3DG_ERR_UNSUPPORTED;
    }
    int launches = 0;
    const int rc = launch_adam(num_tensors, tensors, (cudaStream_t)stream, &launches);
    r3dg_adam_launches += (unsigned long long)launches;
    return rc;
}

}  // extern "C"
