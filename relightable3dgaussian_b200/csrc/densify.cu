// Stage-1 densification (SURVEY.md §8(f)3): the reference's `add_densification_stats` and `densify_and_prune`
// (scene/gaussian_model.py:890-937) as four kernels.  The reference clones, splits and prunes with boolean indexing
// and `torch.cat`, copying every per-Gaussian tensor four times (to P+Kc rows, to P+Kc+2Ks, and through two prunes),
// and every boolean index is a host sync.  Here:
//   densify_stats_kernel     one thread per Gaussian, in place, no host sync;
//   densify_classify_kernel  one read of the statistics, scaling and opacity per row: the row's clone / split
//                            membership and whether each of its (up to four) output rows survives the final prune;
//   block_sums_scan_kernel   7-channel exclusive scan of the per-block counts (scan.cuh, shared with compact.cu);
//   densify_offsets_kernel   per-row destinations in the four output segments;
//   densify_apply_kernel     every final tensor written once, straight from the old one (descriptor table, one
//                            blockIdx.y per tensor, like compact_gather_kernel).
// All of it is HBM-bound by design.  Every comparison and transcendental is the one torch evaluates on the device:
// fp32 thresholds, IEEE division, expf / logf, sigmoid as 1 / (1 + expf(-x)), division by a scalar as a multiply by
// its fp32 reciprocal (torch's CUDA true-divide by a CPU scalar).
#include "common.cuh"
#include "kernels.h"
#include "scan.cuh"

namespace r3dg {

#define DNS_THREADS 256
#define DNS_ITEMS 8
#define DNS_TILE (DNS_THREADS * DNS_ITEMS)
#define DNS_NCH 7

// per-row flag bits (classify) == channel index of the scan
enum { F_KEEP = 0,       // the row itself survives (not split, not pruned)        -> segment A
       F_CLONE_KEEP,     // its clone survives                                       -> segment B
       F_SPLIT_KEEP,     // its two split copies survive                             -> segments C1, C2
       F_SPLIT,          // member of the split set S (rank = normal-sample row)
       F_CLONE,          // member of the clone set C                  (count only)
       F_NORMAL_SEL,     // padded normal gradient >= threshold        (count only, first print)
       F_LIGHT };        // not split, weights_accum < threshold       (count only, second print)

struct DensifyTmp {
    size_t flags, meta, sums, totals, total;
    long long nblocks;
    __host__ DensifyTmp(int P) {
        nblocks = ((long long)P + DNS_TILE - 1) / DNS_TILE;
        const size_t rows = (size_t)(P < 1 ? 1 : P);
        size_t off = 0;
        flags = off;  off = align_up(off + rows, 256);
        meta = off;   off = align_up(off + rows * 16, 256);
        sums = off;   off = align_up(off + (size_t)DNS_NCH * (nblocks + 1) * 4, 256);
        totals = off; off = align_up(off + 8 * 4, 256);
        total = off;
    }
};

__global__ void __launch_bounds__(256) densify_stats_kernel(int P, const float* __restrict__ vgrad, int stride,
                                                            const float* __restrict__ ngrad, const uint8_t* __restrict__ filter,
                                                            const float* __restrict__ weights, const int32_t* __restrict__ radii,
                                                            float* __restrict__ weights_accum, float* __restrict__ xyz_accum,
                                                            float* __restrict__ normal_accum, float* __restrict__ denom,
                                                            float* __restrict__ max_radii2D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    weights_accum[i] += weights[i];
    if (!filter[i]) return;
    const float gx = vgrad[(long long)i * stride], gy = vgrad[(long long)i * stride + 1];
    xyz_accum[i] += sqrtf(gx * gx + gy * gy);
    const float nx = ngrad[3LL * i], ny = ngrad[3LL * i + 1], nz = ngrad[3LL * i + 2];
    normal_accum[i] += sqrtf(nx * nx + ny * ny + nz * nz);
    denom[i] += 1.f;
    if (radii) max_radii2D[i] = fmaxf(max_radii2D[i], (float)radii[i]);
}

// torch.max(dim=1) propagates NaN
__device__ __forceinline__ float max3_nan(float a, float b, float c) {
    float m = (b > a || b != b) ? b : a;
    return (c > m || c != c) ? c : m;
}

__global__ void __launch_bounds__(DNS_THREADS) densify_classify_kernel(int P, const float* __restrict__ xyz_accum,
                                                                       const float* __restrict__ normal_accum,
                                                                       const float* __restrict__ denom,
                                                                       const float* __restrict__ weights_accum,
                                                                       const float* __restrict__ scaling,
                                                                       const float* __restrict__ opacity,
                                                                       const r3dg_densify_thresholds th,
                                                                       uint8_t* __restrict__ flags, uint32_t* __restrict__ sums,
                                                                       long long stride) {
    __shared__ uint32_t s_cnt[DNS_NCH][DNS_THREADS / 32];
    uint32_t cnt[DNS_NCH];
#pragma unroll
    for (int c = 0; c < DNS_NCH; ++c) cnt[c] = 0;
    const long long base = (long long)blockIdx.x * DNS_TILE;
    for (int k = 0; k < DNS_ITEMS; ++k) {
        const long long i = base + (long long)k * DNS_THREADS + threadIdx.x;
        if (i >= P) break;
        const float d = denom[i];
        float g = __fdiv_rn(xyz_accum[i], d), gn = __fdiv_rn(normal_accum[i], d);
        if (g != g) g = 0.f;                                   // only NaN (0/0) becomes 0; x/0 = inf stays
        if (gn != gn) gn = 0.f;
        const float e0 = expf(scaling[3 * i]), e1 = expf(scaling[3 * i + 1]), e2 = expf(scaling[3 * i + 2]);
        const float smax = max3_nan(e0, e1, e2);
        // densify_and_clone takes torch.norm of the [P,1] gradients (sqrt of the square), densify_and_split the raw value
        const float ng = sqrtf(g * g), ngn = sqrtf(gn * gn);
        const bool clone = (ng >= th.max_grad || ngn >= th.max_grad_normal) && smax <= th.dense_scale;
        const bool split = (g >= th.max_grad || gn >= th.max_grad_normal) && smax > th.dense_scale;
        const bool transparent = __fdiv_rn(1.f, 1.f + expf(-opacity[i])) < th.min_opacity;
        // densification_postfix zeroed max_radii2D, so its term is `0 > max_screen_size`
        const bool size_vs = th.check_size && 0.f > th.max_screen_size;
        const bool big = size_vs || (th.check_size && smax > th.big_scale);
        bool big_split = size_vs;
        if (th.check_size && !size_vs && split) {
            const float s0 = expf(logf(__fmul_rn(e0, th.split_recip))), s1 = expf(logf(__fmul_rn(e1, th.split_recip))),
                        s2 = expf(logf(__fmul_rn(e2, th.split_recip)));
            big_split = max3_nan(s0, s1, s2) > th.big_scale;
        }
        const bool new_light = 1.f < th.weights_threshold;     // clones and split copies carry weights_accum = 1
        const bool light = weights_accum[i] < th.weights_threshold;
        uint32_t f = 0;
        f |= (!split && !(transparent || light || big)) ? 1u << F_KEEP : 0u;
        f |= (clone && !(transparent || new_light || big)) ? 1u << F_CLONE_KEEP : 0u;
        f |= (split && !(transparent || new_light || big_split)) ? 1u << F_SPLIT_KEEP : 0u;
        f |= split ? 1u << F_SPLIT : 0u;
        f |= clone ? 1u << F_CLONE : 0u;
        f |= (gn >= th.max_grad_normal) ? 1u << F_NORMAL_SEL : 0u;
        f |= (!split && light) ? 1u << F_LIGHT : 0u;
        flags[i] = (uint8_t)f;
#pragma unroll
        for (int c = 0; c < DNS_NCH; ++c) cnt[c] += (f >> c) & 1u;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < DNS_NCH; ++c) {
        const uint32_t w = __reduce_add_sync(0xffffffffu, cnt[c]);
        if (lane == 0) s_cnt[c][warp] = w;
    }
    __syncthreads();
    if (threadIdx.x < DNS_NCH) {
        uint32_t t = 0;
        for (int w = 0; w < DNS_THREADS / 32; ++w) t += s_cnt[threadIdx.x][w];
        sums[threadIdx.x * stride + blockIdx.x] = t;
    }
}

// Thread t owns DNS_ITEMS consecutive rows, so the in-block order is the row order.  The four scanned channels are
// packed into 16-bit lanes of one u64 (a block counts at most DNS_TILE = 2048 rows per channel).
__global__ void __launch_bounds__(DNS_THREADS) densify_offsets_kernel(int P, const uint8_t* __restrict__ flags,
                                                                      const uint32_t* __restrict__ sums, long long stride,
                                                                      uint4* __restrict__ meta) {
    __shared__ unsigned long long s_warp[DNS_THREADS / 32];
    const long long base = (long long)blockIdx.x * DNS_TILE + (long long)threadIdx.x * DNS_ITEMS;
    // the DNS_ITEMS flag bytes of this thread, row base + k in byte k (rows past P read as 0)
    unsigned long long fl = 0;
    if (base + DNS_ITEMS <= P) {
        fl = *reinterpret_cast<const unsigned long long*>(flags + base);      // base is a multiple of 8
    } else {
        for (int k = 0; k < DNS_ITEMS; ++k)
            if (base + k < P) fl |= (unsigned long long)flags[base + k] << (8 * k);
    }
    unsigned long long c = 0;
#pragma unroll
    for (int k = 0; k < DNS_ITEMS; ++k) {
        const unsigned long long f = (fl >> (8 * k)) & 0xffull;
        c += (f & 1u) | (((f >> 1) & 1u) << 16) | (((f >> 2) & 1u) << 32) | (((f >> 3) & 1u) << 48);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    unsigned long long pre = inc - c;
    for (int w = 0; w < warp; ++w) pre += s_warp[w];
    uint32_t run[4];
#pragma unroll
    for (int ch = 0; ch < 4; ++ch) run[ch] = sums[ch * stride + blockIdx.x] + (uint32_t)((pre >> (16 * ch)) & 0xffffu);
#pragma unroll
    for (int k = 0; k < DNS_ITEMS; ++k) {
        if (base + k >= P) break;
        const uint32_t f = (uint32_t)(fl >> (8 * k));
        const uint32_t b0 = f & 1u, b1 = (f >> 1) & 1u, b2 = (f >> 2) & 1u, b3 = (f >> 3) & 1u;
        meta[base + k] = make_uint4(run[0] | (b0 << 31), run[1] | (b1 << 31), run[2] | (b2 << 31), run[3] | (b3 << 31));
        run[0] += b0; run[1] += b1; run[2] += b2; run[3] += b3;
    }
}

struct DensifyApplyParams {
    long long P, Pn;
    uint32_t totA, totB, totC, nS;
    float split_recip;
    const uint4* meta;
    const float* rot;      // [P,4] old rotations (xyz op)
    const float* scl;      // [P,3] old log-scales (xyz op)
    const float* z;        // [2 nS,3] standard normal samples
    int num;
    r3dg_densify_tensor t[R3DG_DENSIFY_MAX];
};

// Component w of split copy `row` of Gaussian i: build_rotation(q) (normalised) times (z * exp(s)), plus the centre.
// The rotation matrix is rounded op by op as the reference's elementwise expression; the 3x3 product stands in for
// torch.bmm, whose summation order is cuBLAS's.
__device__ __forceinline__ float split_xyz(const DensifyApplyParams& p, long long i, int w, uint32_t row, float x) {
    const float4 r = reinterpret_cast<const float4*>(p.rot)[i];
    const float n = sqrtf(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r.x, r.x), __fmul_rn(r.y, r.y)), __fmul_rn(r.z, r.z)),
                                    __fmul_rn(r.w, r.w)));
    const float qr = __fdiv_rn(r.x, n), qx = __fdiv_rn(r.y, n), qy = __fdiv_rn(r.z, n), qz = __fdiv_rn(r.w, n);
    float R0, R1, R2;
    if (w == 0) {
        R0 = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(__fmul_rn(qy, qy), __fmul_rn(qz, qz))));
        R1 = __fmul_rn(2.f, __fsub_rn(__fmul_rn(qx, qy), __fmul_rn(qr, qz)));
        R2 = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qz), __fmul_rn(qr, qy)));
    } else if (w == 1) {
        R0 = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qy), __fmul_rn(qr, qz)));
        R1 = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qx), __fmul_rn(qz, qz))));
        R2 = __fmul_rn(2.f, __fsub_rn(__fmul_rn(qy, qz), __fmul_rn(qr, qx)));
    } else {
        R0 = __fmul_rn(2.f, __fsub_rn(__fmul_rn(qx, qz), __fmul_rn(qr, qy)));
        R1 = __fmul_rn(2.f, __fadd_rn(__fmul_rn(qy, qz), __fmul_rn(qr, qx)));
        R2 = __fsub_rn(1.f, __fmul_rn(2.f, __fadd_rn(__fmul_rn(qx, qx), __fmul_rn(qy, qy))));
    }
    const float* zr = p.z + 3LL * row;
    const float* s = p.scl + 3 * i;
    const float v0 = __fmul_rn(zr[0], expf(s[0])), v1 = __fmul_rn(zr[1], expf(s[1])), v2 = __fmul_rn(zr[2], expf(s[2]));
    return __fadd_rn(fmaf(R2, v2, fmaf(R1, v1, __fmul_rn(R0, v0))), x);
}

__global__ void __launch_bounds__(256) densify_apply_kernel(const DensifyApplyParams p) {
    const r3dg_densify_tensor t = p.t[blockIdx.y];
    const long long wpr = t.row_bytes >> 2;
    uint32_t* __restrict__ dst = (uint32_t*)t.dst;
    const long long stride = (long long)gridDim.x * blockDim.x;
    if (t.kind == R3DG_DENSIFY_ZERO) {
        for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < p.Pn * wpr; j += stride) dst[j] = 0u;
        return;
    }
    const uint32_t* __restrict__ src = (const uint32_t*)t.src;
    const long long c1 = (long long)p.totA + p.totB, c2 = c1 + p.totC;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < p.P * wpr; j += stride) {
        const long long i = j / wpr;
        const int w = (int)(j - i * wpr);
        const uint4 m = p.meta[i];
        if (!((m.x | m.y | m.z) >> 31)) continue;
        const uint32_t v = src[j];
        if (m.x >> 31) dst[(long long)(m.x & 0x7fffffffu) * wpr + w] = v;
        if (m.y >> 31) dst[((long long)p.totA + (m.y & 0x7fffffffu)) * wpr + w] = t.kind == R3DG_DENSIFY_MOMENT ? 0u : v;
        if (m.z >> 31) {
            const long long o = m.z & 0x7fffffffu;
            uint32_t n1 = v, n2 = v;
            if (t.kind == R3DG_DENSIFY_MOMENT) {
                n1 = n2 = 0u;
            } else if (t.kind == R3DG_DENSIFY_SCALING) {
                n1 = n2 = __float_as_uint(logf(__fmul_rn(expf(__uint_as_float(v)), p.split_recip)));
            } else if (t.kind == R3DG_DENSIFY_XYZ) {
                const uint32_t k = m.w & 0x7fffffffu;
                n1 = __float_as_uint(split_xyz(p, i, w, k, __uint_as_float(v)));
                n2 = __float_as_uint(split_xyz(p, i, w, p.nS + k, __uint_as_float(v)));
            }
            dst[(c1 + o) * wpr + w] = n1;
            dst[(c2 + o) * wpr + w] = n2;
        }
    }
}

size_t densify_tmp_bytes(int P) { return DensifyTmp(P).total; }

int launch_densify_stats(int P, const float* vgrad, int stride, const float* ngrad, const uint8_t* filter, const float* weights,
                         const int32_t* radii, float* weights_accum, float* xyz_accum, float* normal_accum, float* denom,
                         float* max_radii2D, cudaStream_t stream) {
    if (P < 0 || stride < 2) return R3DG_ERR_BAD_ARG;
    if (P == 0) return 0;
    if (!vgrad || !ngrad || !filter || !weights || !weights_accum || !xyz_accum || !normal_accum || !denom) return R3DG_ERR_BAD_ARG;
    if ((radii == nullptr) != (max_radii2D == nullptr)) return R3DG_ERR_BAD_ARG;
    densify_stats_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, vgrad, stride, ngrad, filter, weights, radii, weights_accum,
                                                              xyz_accum, normal_accum, denom, max_radii2D);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_densify_classify(int P, const float* xyz_accum, const float* normal_accum, const float* denom,
                            const float* weights_accum, const float* scaling, const float* opacity,
                            const r3dg_densify_thresholds& th, void* tmp_, size_t tmp_bytes, int* totals_host,
                            cudaStream_t stream) {
    const DensifyTmp t(P);
    if (P < 0 || !tmp_ || tmp_bytes < t.total) return R3DG_ERR_BAD_ARG;
    if (P > 0 && (!xyz_accum || !normal_accum || !denom || !weights_accum || !scaling || !opacity)) return R3DG_ERR_BAD_ARG;
    char* tmp = (char*)tmp_;
    uint32_t* sums = (uint32_t*)(tmp + t.sums);
    uint32_t* totals = (uint32_t*)(tmp + t.totals);
    const long long stride = t.nblocks + 1;
    if (P > 0)
        densify_classify_kernel<<<(unsigned)t.nblocks, DNS_THREADS, 0, stream>>>(P, xyz_accum, normal_accum, denom, weights_accum,
                                                                                 scaling, opacity, th, (uint8_t*)(tmp + t.flags),
                                                                                 sums, stride);
    block_sums_scan_kernel<DNS_NCH><<<1, 1024, 0, stream>>>(P > 0 ? t.nblocks : 0, stride, sums, totals);
    if (P > 0)
        densify_offsets_kernel<<<(unsigned)t.nblocks, DNS_THREADS, 0, stream>>>(P, (const uint8_t*)(tmp + t.flags), sums, stride,
                                                                                (uint4*)(tmp + t.meta));
    if (totals_host) R3DG_CUDA_TRY(cudaMemcpyAsync(totals_host, totals, DNS_NCH * sizeof(int), cudaMemcpyDeviceToHost, stream));
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_densify_apply(int P, const int* totals, int num, const r3dg_densify_tensor* tensors, const float* rotation,
                         const float* scaling, const float* samples, float split_recip, const void* tmp_, size_t tmp_bytes,
                         int num_sms, cudaStream_t stream) {
    const DensifyTmp t(P);
    if (P < 0 || !totals || num < 0 || num > R3DG_DENSIFY_MAX || (num > 0 && !tensors) || !tmp_ || tmp_bytes < t.total)
        return R3DG_ERR_BAD_ARG;
    for (int c = 0; c < DNS_NCH; ++c)
        if (totals[c] < 0 || totals[c] > P) return R3DG_ERR_BAD_ARG;
    const long long Pn = (long long)totals[F_KEEP] + totals[F_CLONE_KEEP] + 2LL * totals[F_SPLIT_KEEP];
    const int nS = totals[F_SPLIT];
    if (Pn > 0x7fffffffLL || totals[F_SPLIT_KEEP] > nS) return R3DG_ERR_BAD_ARG;
    DensifyApplyParams p;
    p.P = P; p.Pn = Pn;
    p.totA = (uint32_t)totals[F_KEEP]; p.totB = (uint32_t)totals[F_CLONE_KEEP]; p.totC = (uint32_t)totals[F_SPLIT_KEEP];
    p.nS = (uint32_t)nS; p.split_recip = split_recip;
    p.meta = (const uint4*)((const char*)tmp_ + t.meta);
    p.rot = rotation; p.scl = scaling; p.z = samples; p.num = num;
    for (int k = 0; k < num; ++k) {
        const r3dg_densify_tensor& d = tensors[k];
        if (d.row_bytes <= 0 || (d.row_bytes & 3) || (!d.dst && Pn > 0) || d.kind < 0 || d.kind > R3DG_DENSIFY_ZERO)
            return R3DG_ERR_BAD_ARG;
        if (d.kind != R3DG_DENSIFY_ZERO && !d.src && P > 0) return R3DG_ERR_BAD_ARG;
        if ((d.kind == R3DG_DENSIFY_XYZ || d.kind == R3DG_DENSIFY_SCALING) && d.row_bytes != 12) return R3DG_ERR_BAD_ARG;
        if (d.kind == R3DG_DENSIFY_XYZ && (!rotation || !scaling || (nS > 0 && !samples))) return R3DG_ERR_BAD_ARG;
        p.t[k] = d;
    }
    if (P == 0 || num == 0) return 0;
    densify_apply_kernel<<<dim3((unsigned)(num_sms * 8), (unsigned)num), 256, 0, stream>>>(p);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
