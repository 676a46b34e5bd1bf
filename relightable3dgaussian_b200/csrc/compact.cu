// §8(f)3, the surgery half: densify-and-prune removes / keeps rows of EVERY per-Gaussian tensor — 7-13 parameters,
// their two Adam moments and four statistics — with one boolean mask (reference scene/gaussian_model.py:682-700
// `_prune_optimizer`, :702-729 `prune_points`, :890-929 `densify_and_prune`): ~40 `tensor[mask]` launches, each
// re-deriving the same prefix sum of the mask.  Here: ONE scan of the mask, then ONE gather launch that moves the kept
// rows of all tensors (descriptor table in the kernel parameters, like adam.cu).  HBM-bound: reads + writes the kept
// bytes once.  Row order is preserved (stable), exactly what boolean indexing gives.
#include "common.cuh"
#include "kernels.h"
#include "scan.cuh"

namespace r3dg {

#define CMP_THREADS 256
#define CMP_ITEMS 8
#define CMP_TILE (CMP_THREADS * CMP_ITEMS)

// layout of tmp: u32 offsets[P] (exclusive), u32 block_sums[nblocks + 1], u32 total
struct CompactTmp {
    size_t offsets, block_sums, total_off, total;
    long long nblocks;
    __host__ CompactTmp(int P) {
        nblocks = ((long long)P + CMP_TILE - 1) / CMP_TILE;
        size_t off = 0;
        offsets = off;    off = align_up(off + (size_t)(P < 1 ? 1 : P) * 4, 256);
        block_sums = off; off = align_up(off + (size_t)(nblocks + 1) * 4, 256);
        total_off = off;  off = align_up(off + 4, 256);
        total = off;
    }
};

__global__ void __launch_bounds__(CMP_THREADS) compact_block_sums_kernel(int P, const uint8_t* __restrict__ keep,
                                                                         uint32_t* __restrict__ block_sums) {
    __shared__ uint32_t s_warp[CMP_THREADS / 32];
    const long long base = (long long)blockIdx.x * CMP_TILE;
    uint32_t c = 0;
    for (int k = 0; k < CMP_ITEMS; ++k) {
        const long long i = base + (long long)k * CMP_THREADS + threadIdx.x;
        if (i < P) c += keep[i] ? 1u : 0u;
    }
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < CMP_THREADS / 32; ++w) t += s_warp[w];
        block_sums[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(CMP_THREADS) compact_offsets_kernel(int P, const uint8_t* __restrict__ keep,
                                                                      const uint32_t* __restrict__ block_sums,
                                                                      uint32_t* __restrict__ offsets) {
    // thread t owns CMP_ITEMS CONSECUTIVE rows so that the in-block order is the row order
    __shared__ uint32_t s_warp[CMP_THREADS / 32];
    const long long base = (long long)blockIdx.x * CMP_TILE + (long long)threadIdx.x * CMP_ITEMS;
    uint32_t f[CMP_ITEMS], c = 0;
#pragma unroll
    for (int k = 0; k < CMP_ITEMS; ++k) { f[k] = (base + k < P && keep[base + k]) ? 1u : 0u; c += f[k]; }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    uint32_t run = block_sums[blockIdx.x] + inc - c;
    for (int w = 0; w < warp; ++w) run += s_warp[w];
#pragma unroll
    for (int k = 0; k < CMP_ITEMS; ++k)
        if (base + k < P) { offsets[base + k] = run; run += f[k]; }
}

struct CompactParams {
    int P, num;
    const uint8_t* keep;
    const uint32_t* offsets;
    r3dg_compact_tensor t[R3DG_COMPACT_MAX];
};

// blockIdx.y = tensor; each thread moves 4-byte words of kept rows (rows are 4..192 B: consecutive threads cover
// consecutive words of consecutive rows, so both sides stay coalesced)
__global__ void __launch_bounds__(256) compact_gather_kernel(const CompactParams p) {
    const r3dg_compact_tensor t = p.t[blockIdx.y];
    const long long wpr = t.row_bytes >> 2;
    const long long total = (long long)p.P * wpr;
    const uint32_t* __restrict__ src = (const uint32_t*)t.src;
    uint32_t* __restrict__ dst = (uint32_t*)t.dst;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / wpr, w = i - row * wpr;
        if (p.keep[row]) dst[(long long)p.offsets[row] * wpr + w] = src[i];
    }
}

size_t compact_tmp_bytes(int P) { return CompactTmp(P).total; }

int launch_compact_scan(int P, const uint8_t* keep, void* tmp_, size_t tmp_bytes, int* count_host, cudaStream_t stream) {
    const CompactTmp t(P);
    if (tmp_bytes < t.total) return R3DG_ERR_BAD_ARG;
    char* tmp = (char*)tmp_;
    uint32_t* sums = (uint32_t*)(tmp + t.block_sums);
    uint32_t* total = (uint32_t*)(tmp + t.total_off);
    if (P > 0) compact_block_sums_kernel<<<(unsigned)t.nblocks, CMP_THREADS, 0, stream>>>(P, keep, sums);
    block_sums_scan_kernel<1><<<1, 1024, 0, stream>>>(P > 0 ? t.nblocks : 0, 0, sums, total);
    if (P > 0) compact_offsets_kernel<<<(unsigned)t.nblocks, CMP_THREADS, 0, stream>>>(P, keep, sums, (uint32_t*)(tmp + t.offsets));
    if (count_host) R3DG_CUDA_TRY(cudaMemcpyAsync(count_host, total, sizeof(int), cudaMemcpyDeviceToHost, stream));
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_compact_rows(int P, int num, const r3dg_compact_tensor* tensors, const uint8_t* keep, const void* tmp_,
                        int num_sms, cudaStream_t stream) {
    if (P <= 0 || num <= 0) return 0;
    const CompactTmp t(P);
    for (int k0 = 0; k0 < num; k0 += R3DG_COMPACT_MAX) {
        CompactParams p;
        p.P = P; p.keep = keep; p.offsets = (const uint32_t*)((const char*)tmp_ + t.offsets);
        p.num = num - k0 < R3DG_COMPACT_MAX ? num - k0 : R3DG_COMPACT_MAX;
        for (int k = 0; k < p.num; ++k) {
            p.t[k] = tensors[k0 + k];
            if (p.t[k].row_bytes <= 0 || (p.t[k].row_bytes & 3) || !p.t[k].src || !p.t[k].dst) return R3DG_ERR_BAD_ARG;
        }
        compact_gather_kernel<<<dim3((unsigned)(num_sms * 8), (unsigned)p.num), 256, 0, stream>>>(p);
    }
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
