// Stable LSD radix sort of (u32 key, u32 value) pairs.  In the rasterizer it orders the Gaussians
// by view depth once (P pairs) instead of the reference's cub::DeviceRadixSort::SortPairs over
// all R ~ 8 P (tile, depth) instances (rasterizer_impl.cu:313-318); the per-tile lists are then
// produced by the order-preserving binning in binning.cu.  The BVH and kNN builders sort their
// 30-bit Morton codes with it (bvh.cu, knn.cu).  Hand-written for sm_90a:
//
//   sort_histogram_kernel : per-tile digit counts of the first pass;
//   per pass:
//   sort_tilescan_kernel  : per digit, exclusive prefix of the per-tile counts over the tiles
//                           (one warp per digit, digit-major planes) and the digit's total (= the
//                           pass's global histogram); clears the count plane of the next pass;
//   sort_scatter_kernel   : one CTA per 2048-pair tile: stable ranking (per-warp ballot matching),
//                           destination = digit base + tile prefix + rank, reorder through shared
//                           memory so that global writes are digit-contiguous runs; while it
//                           writes a pair it already counts it for the NEXT pass
//                           (count[destination tile][next digit] += 1, one global reduction).
//
// An earlier version chained the tiles with a decoupled look-back (one kernel per pass).  The sorts
// here are small (P ~ 1M pairs = ~500 tiles, all resident at once), so every tile had to poll
// hundreds of predecessors' descriptors, and most of each pass was spent polling.  Counting ahead removes every inter-CTA wait: nothing spins, nothing can deadlock.
//
// Which key bits need sorting is decided on the device (sort_plan in common.cuh): no host sync.
#include <algorithm>
#include "common.cuh"
#include "kernels.h"

namespace r3dg {

constexpr int SORT_NW = R3DG_SORT_THREADS / 32;
constexpr int SORT_PER_WARP = R3DG_SORT_TILE / SORT_NW;      // 256 consecutive pairs per warp

__global__ void __launch_bounds__(R3DG_SORT_THREADS) sort_histogram_kernel(GeomHeader* __restrict__ header, long long n,
                                                                           const uint32_t* __restrict__ keys,
                                                                           uint32_t* __restrict__ tilecnt0, long long tstride) {
    __shared__ uint32_t th[256];                             // first-pass digit counts of the current tile
    int passes, w;
    sort_plan(header->depth_or & header->depth_nor, passes, w);
    if (blockIdx.x == 0 && threadIdx.x == 0) header->sort_exec = (uint32_t)passes;
    if (passes == 0) return;
    const uint32_t mask = (1u << w) - 1u;
    const long long ntiles = (n + R3DG_SORT_TILE - 1) / R3DG_SORT_TILE;
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        __syncthreads();
        th[threadIdx.x] = 0;
        __syncthreads();
        const long long base = tile * R3DG_SORT_TILE;
#pragma unroll
        for (int i = 0; i < R3DG_SORT_ITEMS; ++i) {
            const long long j = base + i * R3DG_SORT_THREADS + threadIdx.x;
            if (j < n) atomicAdd(&th[keys[j] & mask], 1u);
        }
        __syncthreads();
        tilecnt0[(size_t)threadIdx.x * tstride + tile] = th[threadIdx.x];
    }
}

// Count planes are digit-major, cnt[digit][tile] (row pitch tstride): the scan direction is contiguous.
// grid = 32 CTAs x 8 warps, warp <-> digit: exclusive prefix over the tiles in place, the digit's
// total -> hist[slot][digit] (the pass's global histogram), and the next pass's plane is cleared.
__global__ void __launch_bounds__(256) sort_tilescan_kernel(const GeomHeader* __restrict__ header, long long n, int slot,
                                                            uint32_t* __restrict__ cnt, uint32_t* __restrict__ cnt_next,
                                                            long long tstride, uint32_t* __restrict__ hist) {
    int passes, w;
    sort_plan(header->depth_or & header->depth_nor, passes, w);
    if (slot >= passes) return;
    const int lane = threadIdx.x & 31, d = blockIdx.x * 8 + (threadIdx.x >> 5);
    const long long ntiles = (n + R3DG_SORT_TILE - 1) / R3DG_SORT_TILE;
    uint32_t* row = cnt + (size_t)d * tstride;
    uint32_t* nrow = cnt_next + (size_t)d * tstride;
    uint32_t carry = 0;
    for (long long t0 = 0; t0 < ntiles; t0 += 256) {         // 8 independent coalesced loads in flight per lane
        uint32_t v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { const long long t = t0 + j * 32 + lane; v[j] = t < ntiles ? row[t] : 0u; }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const long long t = t0 + j * 32 + lane;
            uint32_t inc = v[j];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
            if (t < ntiles) { row[t] = carry + inc - v[j]; nrow[t] = 0u; }
            carry += __shfl_sync(0xffffffffu, inc, 31);
        }
    }
    if (lane == 0) hist[slot * 256 + d] = carry;
}

struct SortSmem {
    uint32_t keys[R3DG_SORT_TILE];
    uint32_t vals[R3DG_SORT_TILE];
    uint32_t warp_hist[SORT_NW][256];
    uint32_t local_off[256];     // exclusive prefix of the digit counts inside the tile
    uint32_t global_off[256];    // global start of this tile's run of digit d
    uint32_t s_w[SORT_NW];
};

__global__ void __launch_bounds__(R3DG_SORT_THREADS, 4) sort_scatter_kernel(
    const GeomHeader* __restrict__ header, long long n, int slot, const uint32_t* __restrict__ keys_in,
    const uint32_t* __restrict__ vals_in, uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out,
    const uint32_t* __restrict__ hist, const uint32_t* __restrict__ tile_prefix, uint32_t* __restrict__ cnt_next,
    long long tstride) {
    __shared__ SortSmem sm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int passes, w;
    sort_plan(header->depth_or & header->depth_nor, passes, w);
    if (slot >= passes) return;                          // fewer digits needed than slots launched
    const int shift = slot * w;
    const uint32_t mask = (1u << w) - 1u;
    const bool count_next = slot + 1 < passes;
    const long long ntiles = (n + R3DG_SORT_TILE - 1) / R3DG_SORT_TILE;

    // global start of digit tid: exclusive scan of this pass's histogram (thread d <-> digit d)
    uint32_t digit_base;
    {
        const uint32_t hv = hist[slot * 256 + tid];
        uint32_t inc = hv;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t t2 = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t2; }
        if (lane == 31) sm.s_w[warp] = inc;
        __syncthreads();
        uint32_t woff = 0;
#pragma unroll
        for (int ww = 0; ww < SORT_NW; ++ww) if (ww < warp) woff += sm.s_w[ww];
        digit_base = woff + inc - hv;
    }

    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        __syncthreads();
        for (int i = tid; i < SORT_NW * 256; i += R3DG_SORT_THREADS) (&sm.warp_hist[0][0])[i] = 0;
        const uint32_t tp = tile_prefix[(size_t)tid * tstride + tile];     // requested early
        __syncthreads();
        const long long tile_base = tile * R3DG_SORT_TILE;
        const int count = (int)min((long long)R3DG_SORT_TILE, n - tile_base);

        // ---- load + stable ranking within the warp's 256-pair slice -------------------------------
        uint32_t k[R3DG_SORT_ITEMS], v[R3DG_SORT_ITEMS], dg[R3DG_SORT_ITEMS], rank[R3DG_SORT_ITEMS];
#pragma unroll
        for (int i = 0; i < R3DG_SORT_ITEMS; ++i) {
            const int local = warp * SORT_PER_WARP + i * 32 + lane;
            const bool valid = local < count;
            k[i] = valid ? keys_in[tile_base + local] : 0u;
            v[i] = valid ? vals_in[tile_base + local] : 0u;
            // padding slots take the last digit: they trail every valid key (they are the tail of the tile),
            // so valid ranks are unaffected, and they are never stored
            dg[i] = valid ? ((k[i] >> shift) & mask) : mask;
        }
#pragma unroll
        for (int i = 0; i < R3DG_SORT_ITEMS; ++i) {
            // peers with the same digit, from w ballots rather than one match.any over ~32 distinct values
            // (tools/ubench.cu measures both)
            uint32_t peers = 0xffffffffu;
#pragma unroll
            for (int b = 0; b < 8; ++b) {
                if (b < w) {
                    const bool bit = (dg[i] >> b) & 1u;
                    const uint32_t m = __ballot_sync(0xffffffffu, bit);
                    peers &= bit ? m : ~m;
                }
            }
            const int leader = __ffs(peers) - 1;
            const uint32_t below = __popc(peers & ((1u << lane) - 1u));
            uint32_t old = 0;
            if (lane == leader) { old = sm.warp_hist[warp][dg[i]]; sm.warp_hist[warp][dg[i]] = old + __popc(peers); }
            old = __shfl_sync(0xffffffffu, old, leader);
            rank[i] = old + below;
            __syncwarp();
        }
        __syncthreads();

        // ---- per digit (thread d <-> digit d): warp prefixes, tile-local and global offsets ------------
        {
            const int d = tid;
            uint32_t acc = 0;
#pragma unroll
            for (int ww = 0; ww < SORT_NW; ++ww) { const uint32_t t = sm.warp_hist[ww][d]; sm.warp_hist[ww][d] = acc; acc += t; }
            // the padding of the last tile was counted under digit `mask`; it sits behind every valid key,
            // so only the total of that (last) digit is inflated, which nothing reads
            uint32_t inc = acc;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { uint32_t t2 = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t2; }
            if (lane == 31) sm.s_w[warp] = inc;
            __syncthreads();
            uint32_t woff = 0;
#pragma unroll
            for (int ww = 0; ww < SORT_NW; ++ww) if (ww < warp) woff += sm.s_w[ww];
            sm.local_off[d] = woff + inc - acc;
            sm.global_off[d] = digit_base + tp;
        }
        __syncthreads();

        // ---- reorder through shared memory, then digit-contiguous global writes ----------------------
#pragma unroll
        for (int i = 0; i < R3DG_SORT_ITEMS; ++i) {
            const bool valid = warp * SORT_PER_WARP + i * 32 + lane < count;
            if (valid) {
                const uint32_t pos = sm.local_off[dg[i]] + sm.warp_hist[warp][dg[i]] + rank[i];
                sm.keys[pos] = k[i];
                sm.vals[pos] = v[i];
            }
        }
        __syncthreads();
        for (int i = tid; i < count; i += R3DG_SORT_THREADS) {
            const uint32_t kk = sm.keys[i];
            const uint32_t dd = (kk >> shift) & mask;
            const uint32_t dst = sm.global_off[dd] + ((uint32_t)i - sm.local_off[dd]);
            keys_out[dst] = kk;
            vals_out[dst] = sm.vals[i];
            // count the pair for the next pass at its new position
            if (count_next) atomicAdd(&cnt_next[(size_t)((kk >> (shift + w)) & mask) * tstride + dst / R3DG_SORT_TILE], 1u);
        }
    }
}

// header: depth_or / depth_nor hold the OR of the keys and of their complements.  On return
// (stream order) the sorted pairs are in buffer (header->sort_exec & 1).
int launch_sort(void* geom_header, char* buf, const SortLayout& sl, long long n, int num_sms,
                cudaStream_t stream) {
    if (n > sl.n || n >= (1ll << 30)) return R3DG_ERR_BAD_ARG;
    GeomHeader* header = (GeomHeader*)geom_header;
    uint32_t* hist = (uint32_t*)(buf + sl.hist);
    uint32_t* c0 = (uint32_t*)(buf + sl.tilecnt);
    uint32_t* c1 = c0 + (size_t)sl.plane_words;
    const long long ntiles = (n + R3DG_SORT_TILE - 1) / R3DG_SORT_TILE;
    const int grid = (int)std::min<long long>((long long)num_sms * 8, std::max<long long>(1, ntiles));
    sort_histogram_kernel<<<grid, R3DG_SORT_THREADS, 0, stream>>>(header, n, (const uint32_t*)(buf + sl.keys_a), c0, sl.tiles);
    uint32_t* ka = (uint32_t*)(buf + sl.keys_a); uint32_t* kb = (uint32_t*)(buf + sl.keys_b);
    uint32_t* va = (uint32_t*)(buf + sl.vals_a); uint32_t* vb = (uint32_t*)(buf + sl.vals_b);
    for (int k = 0; k < R3DG_SORT_MAX_PASSES; ++k) {
        const bool even = (k & 1) == 0;
        sort_tilescan_kernel<<<32, 256, 0, stream>>>(header, n, k, even ? c0 : c1, even ? c1 : c0, sl.tiles, hist);
        sort_scatter_kernel<<<grid, R3DG_SORT_THREADS, 0, stream>>>(
            header, n, k, even ? ka : kb, even ? va : vb, even ? kb : ka, even ? vb : va, hist,
            even ? c0 : c1, even ? c1 : c0, sl.tiles);
    }
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
