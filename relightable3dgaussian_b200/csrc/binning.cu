// Depth-ordered tile binning: builds the per-tile, depth-sorted Gaussian lists
// (binningState.point_list + imgState.ranges) that the reference obtains from
// duplicateWithKeys -> cub::DeviceRadixSort::SortPairs over 64-bit (tile | depth) keys ->
// identifyTileRanges (rasterizer_impl.cu:70-138, 296-333).
//
// The reference sorts all R ~ 8 P (tile, Gaussian) instances by (tile, depth), stable, instances
// emitted in Gaussian-index order.  The same total order is obtained much cheaper:
//   1. stable-sort the P Gaussians by their depth bits (radix_sort.cu; ties keep index order);
//   2. append them, in that order, to the lists of the tiles their rectangle covers.
// Step 2 is a counting sort by tile id that must preserve the sequence order, done with two
// passes over the depth-sorted sequence cut into chunks (one CTA per chunk, per-tile tables in
// shared memory):
//   bin_count                  : M[chunk][tile] = number of instances the chunk adds to the tile;
//   bin_colsum(+starts)/apply  : exclusive scan of every column of M (per tile over the chunks),
//                                exclusive scan of the tile totals -> ranges[tile], R, and the
//                                compositors' tile order; M becomes the absolute first slot of
//                                (chunk, tile), row M[chunks] the end of every tile's list;
//   bin_scatter                : every chunk takes its per-tile counts from two rows of M, re-walks its
//                                Gaussians and writes each instance to M[chunk][tile] + (rank inside
//                                the chunk, in sequence order), with its block mask and a zeroed
//                                contributor mask.
// Equal (tile, depth) keys end up in Gaussian-index order, exactly as the reference's stable sort
// leaves them, so point_list and ranges are bit-identical.
#include <algorithm>
#include <cstdlib>
#include "common.cuh"
#include "kernels.h"

namespace r3dg {

// bin_count: one CTA per chunk, one thread per Gaussian walking its own rectangle; counting
// needs no order, so the lanes work on different Gaussians in parallel with fire-and-forget
// shared atomics on the CTA's table.
#define BIN_COUNT_THREADS 512       // the grid is one CTA per chunk, fewer than 4 per SM at the headline
__global__ void __launch_bounds__(BIN_COUNT_THREADS) bin_count_kernel(int P, int T, int gx, int CH,
                                                        const GeomHeader* __restrict__ header,
                                                        const uint32_t* __restrict__ vals_a,
                                                        const uint32_t* __restrict__ vals_b,
                                                        const uint2* __restrict__ rects, uint32_t* __restrict__ M) {
    extern __shared__ __align__(16) uint32_t bin_smem[];
    uint32_t* tbl = bin_smem;
    const uint32_t* __restrict__ order = (header->sort_exec & 1u) ? vals_b : vals_a;
    const int c = blockIdx.x;
    const int j0 = c * CH, j1 = min(P, j0 + CH);
    for (int t = threadIdx.x; t < T; t += blockDim.x) tbl[t] = 0u;
    __syncthreads();
    for (int j = j0 + threadIdx.x; j < j1; j += blockDim.x) {
        const uint2 r = rects[order[j]];
        const uint32_t w = r.y & 0xffffu, h = r.y >> 16;
        // one flat loop over the w*h tiles (lanes have different rectangles: nested loops would
        // serialise max(h) * max(w) trips per warp instead of max(w*h))
        uint32_t tile = (r.x >> 16) * (uint32_t)gx + (r.x & 0xffffu), x = 0;
        const uint32_t n = w * h, skip = (uint32_t)gx - w;
#pragma unroll 1
        for (uint32_t k = 0; k < n; ++k) {
            atomicAdd(&tbl[tile], 1u);
            ++tile;
            if (++x == w) { x = 0; tile += skip; }
        }
    }
    __syncthreads();
    uint32_t* row = M + (size_t)c * T;
    for (int t = threadIdx.x; t < T; t += blockDim.x) row[t] = tbl[t];
}

// bin_scatter: one CTA per chunk.  Writing every instance straight to its slot costs one 4-byte
// L2 write transaction per instance (~8M scattered sector writes at the headline config, whatever
// the ranking logic).  Instead the chunk's instances are first gathered in shared memory grouped by tile:
//   1. per-tile counts of the chunk = M[chunk + 1][tile] - M[chunk][tile] (bin_apply left the absolute
//      first slots there, and the list ends in the row after the last chunk), exclusive scan -> local
//      CSR offsets;
//   2. unordered append: one thread per Gaussian, slot = shared atomicAdd on the tile's cursor,
//      entry = tile << 16 | position in the chunk (4 bytes); the Gaussian's id and block rectangle
//      are staged once per position;
//   3. one thread per staged entry: rank = number of entries of its run (same tile) that come
//      earlier in the sequence; global slot = M[chunk][tile] + rank.  A warp's lanes hold
//      consecutive staged entries, i.e. whole runs, whose global slots are contiguous: the
//      stores (id, block mask byte, zeroed contributor mask byte) coalesce into a few sectors per
//      run instead of one transaction per entry.
// A chunk whose instances exceed the staging area is handled in several windows of tiles.
#define BIN_SCATTER_THREADS 1024
#define BIN_LONG_RUN 24            // runs longer than this are ranked through the bitmap
#define BIN_MAX_LONG 2048          // >= staging capacity / BIN_LONG_RUN

// t / gx for t, gx < 2^16 as a multiply-high: gx_inv = 2^32 / gx + 1 (exact, the error stays below 2^-16 < 1 / gx)
__device__ __forceinline__ uint32_t tile_row(int t, unsigned long long gx_inv) {
    return (uint32_t)(((unsigned long long)(uint32_t)t * gx_inv) >> 32);
}

__global__ void __launch_bounds__(BIN_SCATTER_THREADS) bin_scatter_kernel(
    int P, int T, int gx, unsigned long long gx_inv, int CH, int cap, const GeomHeader* __restrict__ header,
    const uint32_t* __restrict__ vals_a,
    const uint32_t* __restrict__ vals_b, const uint2* __restrict__ rects, const uint2* __restrict__ brects,
    const uint32_t* __restrict__ M, uint32_t* __restrict__ point_list, uint8_t* __restrict__ bmask,
    uint8_t* __restrict__ cmask, long long capacity, int starts_in_smem, uint32_t row_base) {
    extern __shared__ __align__(16) uint32_t bin_smem[];
    const size_t T4 = ((size_t)T + 3) & ~(size_t)3;
    uint32_t* a = bin_smem;                               // [T] counts -> exclusive offsets -> cursors
    uint32_t* s_start = bin_smem + T4;                    // [T] (if it fits) copy of the chunk's row of M
    const int words = (CH + 31) >> 5;                     // bitmap over the chunk positions, per warp
    uint32_t* bitmaps = s_start + (starts_in_smem ? T4 : 0);
    uint32_t* s_id = bitmaps + (size_t)(BIN_SCATTER_THREADS / 32) * 2 * words;     // [CH] Gaussian id per position
    uint2* s_br = reinterpret_cast<uint2*>(s_id + CH);                             // [CH] its block rectangle
    uint32_t* stage = reinterpret_cast<uint32_t*>(s_br + CH);                      // [cap] tile << 16 | position
    __shared__ uint32_t s_warp[BIN_SCATTER_THREADS / 32];
    __shared__ int s_hi;
    __shared__ uint32_t s_total, s_nlong;
    __shared__ uint16_t s_long[BIN_MAX_LONG];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t* __restrict__ order = (header->sort_exec & 1u) ? vals_b : vals_a;
    const int c = blockIdx.x;
    const int j0 = c * CH, j1 = min(P, j0 + CH);
    const uint32_t* __restrict__ row = M + (size_t)c * T;
    // ---- 1. per-tile counts of the chunk, exclusive scan over the tiles --------------------------
    for (int t = tid; t < T; t += BIN_SCATTER_THREADS) {
        const uint32_t s = row[t];
        a[t] = row[T + t] - s;
        if (starts_in_smem) s_start[t] = s;
    }
    // the first global slot of (chunk, tile) for step 3: from shared memory when the table fits, else from L2
    const uint32_t* start = starts_in_smem ? s_start : row;
    __syncthreads();
    const int per = (T + BIN_SCATTER_THREADS - 1) / BIN_SCATTER_THREADS;
    const int t0 = min(T, tid * per), t1 = min(T, t0 + per);
    uint32_t sum = 0;
    for (int t = t0; t < t1; ++t) sum += a[t];
    uint32_t inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        const uint32_t wv = lane < BIN_SCATTER_THREADS / 32 ? s_warp[lane] : 0u;
        uint32_t wi = wv;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += v; }
        if (lane < BIN_SCATTER_THREADS / 32) s_warp[lane] = wi - wv;
        if (lane == 31) s_total = wi;
    }
    __syncthreads();
    {
        uint32_t run = s_warp[warp] + inc - sum;
        for (int t = t0; t < t1; ++t) { const uint32_t n = a[t]; a[t] = run; run += n; }     // a[t] = first local slot of tile t
    }
    __syncthreads();
    // ---- windows of tiles whose instances fit the staging area (normally a single one) ------------
    int lo = 0;
    while (lo < T) {
        if (tid == 0) {
            // E(t) = first local slot of tile t (a[] is still pristine for tiles >= lo), E(T) = total.
            // Largest hi in (lo, T] with E(hi) - E(lo) <= cap; one tile never exceeds CH <= cap entries.
            const uint32_t limit = a[lo] + (uint32_t)cap;
            int l = T;
            if (s_total > limit) {
                l = lo + 1;
                int h = T - 1;
                while (l < h) { const int mid = (l + h + 1) >> 1; if (a[mid] <= limit) l = mid; else h = mid - 1; }
            }
            s_hi = l;
        }
        __syncthreads();
        const int hi = s_hi;
        const uint32_t first = a[lo];                      // read before any cursor of this window moves
        if (tid == 0) s_nlong = 0u;
        __syncthreads();
        // ---- 2. unordered append of the window's instances --------------------------------------
        for (int j = j0 + tid; j < j1; j += BIN_SCATTER_THREADS) {
            const uint32_t seq = (uint32_t)(j - j0);
            uint32_t g;
            if (lo == 0) {
                g = order[j];
                s_id[seq] = g;
                s_br[seq] = brects[g];
            } else {
                g = s_id[seq];
            }
            const uint2 r = rects[g];
            // one flat loop over the w*h tiles (lanes have different rectangles: nested loops would
            // serialise max(h) * max(w) trips per warp instead of max(w*h))
            const uint32_t w = r.y & 0xffffu, h = r.y >> 16;
            uint32_t tile = (r.x >> 16) * (uint32_t)gx + (r.x & 0xffffu), x = 0;
            const uint32_t n = w * h, skip = (uint32_t)gx - w;
#pragma unroll 1
            for (uint32_t k = 0; k < n; ++k) {
                if ((int)tile >= lo && (int)tile < hi) {
                    const uint32_t slot = atomicAdd(&a[tile], 1u) - first;
                    stage[slot] = (tile << 16) | seq;
                }
                ++tile;
                if (++x == w) { x = 0; tile += skip; }
            }
        }
        __syncthreads();
        // now a[t] = first slot of tile t+1 for t in [lo, hi)
        const uint32_t n_stage = a[hi - 1] - first;
        // the tiles with a long run (at most n_stage / BIN_LONG_RUN of them)
        for (int t = lo + tid; t < hi; t += BIN_SCATTER_THREADS) {
            const uint32_t rb = (t > lo ? a[t - 1] : first), re = a[t];
            if (re - rb > BIN_LONG_RUN) s_long[atomicAdd(&s_nlong, 1u)] = (uint16_t)t;
        }
        __syncthreads();
        // ---- 3. rank inside the run, coalesced copy-out -------------------------------------------
        // 3a. short runs: one thread per staged entry, all-pairs rank
        for (uint32_t i = tid; i < n_stage; i += BIN_SCATTER_THREADS) {
            const uint32_t e = stage[i];
            const int t = (int)(e >> 16);
            const uint32_t rb = (t > lo ? a[t - 1] : first) - first, re = a[t] - first;
            if (re - rb > BIN_LONG_RUN) continue;
            const uint32_t base = start[t];               // issued before the rank loop, which hides its latency
            uint32_t rank = 0;                            // the run shares the tile: compare whole entries
#pragma unroll 2
            for (uint32_t k = rb; k < re; ++k) rank += (stage[k] < e) ? 1u : 0u;
            const long long pos = (long long)base + rank;
            if (pos < capacity) {
                const uint32_t seq = e & 0xffffu;
                point_list[pos] = row_base + s_id[seq];                 // the view's rows start at row_base
                const uint32_t ty = tile_row(t, gx_inv);
                bmask[pos] = (uint8_t)block_mask_of_rect(s_br[seq], 2u * ((uint32_t)t - ty * (uint32_t)gx), 4u * ty);
                cmask[pos] = 0;
            }
        }
        // 3b. long runs (depth slices that pile up on few tiles): one warp per run; a bitmap over the
        //     chunk positions turns the rank into a prefix population count
        {
            uint32_t* bm = bitmaps + (size_t)warp * 2 * words;     // bits, then the exclusive prefix per word
            uint32_t* bp = bm + words;
            for (uint32_t li = warp; li < s_nlong; li += BIN_SCATTER_THREADS / 32) {
                const int t = (int)s_long[li];
                const uint32_t rb = (t > lo ? a[t - 1] : first) - first, re = a[t] - first;
                for (int k = lane; k < words; k += 32) bm[k] = 0u;
                __syncwarp();
#pragma unroll 1
                for (uint32_t k = rb + lane; k < re; k += 32) { const uint32_t sq = stage[k] & 0xffffu; atomicOr(&bm[sq >> 5], 1u << (sq & 31u)); }
                __syncwarp();
                uint32_t carry = 0;
#pragma unroll 1
                for (int k0 = 0; k0 < words; k0 += 32) {
                    const uint32_t c = (k0 + lane < words) ? (uint32_t)__popc(bm[k0 + lane]) : 0u;
                    uint32_t inc = c;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
                    if (k0 + lane < words) bp[k0 + lane] = carry + inc - c;
                    carry += __shfl_sync(0xffffffffu, inc, 31);
                }
                __syncwarp();
                const uint32_t base = start[t];
                const uint32_t ty = tile_row(t, gx_inv);
                const uint32_t c0 = 2u * ((uint32_t)t - ty * (uint32_t)gx), r0 = 4u * ty;
#pragma unroll 1
                for (uint32_t k = rb + lane; k < re; k += 32) {
                    const uint32_t sq = stage[k] & 0xffffu;
                    const uint32_t rank = bp[sq >> 5] + (uint32_t)__popc(bm[sq >> 5] & ((1u << (sq & 31u)) - 1u));
                    const long long pos = (long long)base + rank;
                    if (pos < capacity) {
                        point_list[pos] = row_base + s_id[sq];
                        bmask[pos] = (uint8_t)block_mask_of_rect(s_br[sq], c0, r0);
                        cmask[pos] = 0;
                    }
                }
                __syncwarp();
            }
        }
        __syncthreads();
        lo = hi;
    }
}

// ---- column scan of M ------------------------------------------------------------------------
// CTA = 32 tiles x 32 groups of BIN_G consecutive chunks (a "slab" of 32*BIN_G chunks);
// grid = (tiles / 32, slabs).
//   bin_colsum  : slab_sum[slab][tile] = sum of the slab's rows; the CTA that finishes last then runs
//   bin_starts  : exclusive scan of the tile totals -> ranges, R; per slab and tile the absolute first
//                 slot (tile start + earlier slabs) -> slab_sum in place; then the compositors' tile
//                 order from the ranges it has just written;
//   bin_apply   : every thread keeps its BIN_G counts in registers, the CTA scans the 32 group sums
//                 through shared memory and M is rewritten as ABSOLUTE first slots; row M[chunks]
//                 receives the end of every tile's list (not clamped to the capacity).
#define BIN_G 16
#define BIN_SLAB (32 * BIN_G)

__device__ __forceinline__ void bin_starts_cta(int T, int slabs, uint32_t* __restrict__ slab_sum, uint2* ranges,
                                               GeomHeader* header, const GeomHeader* prev, long long capacity,
                                               uint32_t* __restrict__ tile_order, uint32_t* __restrict__ bwd_work,
                                               volatile int* count_host);

__global__ void __launch_bounds__(1024) bin_colsum_kernel(int T, int chunks, int slabs, const uint32_t* __restrict__ M,
                                                          uint32_t* __restrict__ slab_sum, uint2* ranges, GeomHeader* header,
                                                          const GeomHeader* prev, long long capacity,
                                                          uint32_t* __restrict__ tile_order, uint32_t* __restrict__ bwd_work,
                                                          volatile int* count_host) {
    __shared__ uint32_t s[32][33];
    __shared__ bool s_last;
    const int tx = threadIdx.x, gy = threadIdx.y;
    const int t = blockIdx.x * 32 + tx;
    const int c0 = blockIdx.y * BIN_SLAB + gy * BIN_G;
    uint32_t sum = 0;
    if (t < T) {
#pragma unroll
        for (int i = 0; i < BIN_G; ++i) if (c0 + i < chunks) sum += M[(size_t)(c0 + i) * T + t];
    }
    s[gy][tx] = sum;
    __syncthreads();
    if (gy == 0) {
        uint32_t acc = 0;
#pragma unroll
        for (int g = 0; g < 32; ++g) acc += s[g][tx];
        if (t < T) slab_sum[(size_t)blockIdx.y * T + t] = acc;
    }
    // the CTA that finishes last runs bin_starts (threadfence-reduction pattern: publish, then take a ticket)
    __threadfence();
    __syncthreads();
    if (tx == 0 && gy == 0) s_last = atomicAdd(&header->bin_ticket, 1u) == gridDim.x * gridDim.y - 1;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    bin_starts_cta(T, slabs, slab_sum, ranges, header, prev, capacity, tile_order, bwd_work, count_host);
}

// Longest-processing-time-first order of the tiles for the compositors: the CTAs of the heavy
// tiles (longest sorted lists) are launched first so that the grid's tail consists of light tiles
// (with row-major order the last heavy CTAs leave SMs idle at the end of the grid).  Coarse counting sort
// by list length (64 buckets), by one CTA of 1024 threads once `ranges` is complete and visible to it.
// Also zeroes bwd_work, which the forward compositor atomicMax-es into.
__device__ __forceinline__ void tile_order_cta(int T, const uint2* ranges, uint32_t* __restrict__ order,
                                               uint32_t* __restrict__ bwd_work) {
    __shared__ uint32_t s_max, s_cnt[64], s_cur[64];
    const int tid = threadIdx.x + blockDim.x * threadIdx.y;
    for (int i = tid; i < 2 * T; i += 1024) bwd_work[i] = 0u;
    if (tid == 0) s_max = 0;
    if (tid < 64) s_cnt[tid] = 0;
    __syncthreads();
    uint32_t m = 0;
    for (int t = tid; t < T; t += 1024) { const uint2 r = ranges[t]; m = max(m, r.y - r.x); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) atomicMax(&s_max, m);
    __syncthreads();
    const uint32_t mx = s_max;
    const int shift = mx < 64 ? 0 : (32 - __clz(mx)) - 6;            // bucket = len >> shift in [0, 63]
    for (int t = tid; t < T; t += 1024) { const uint2 r = ranges[t]; atomicAdd(&s_cnt[min(63u, (r.y - r.x) >> shift)], 1u); }
    __syncthreads();
    if (tid < 32) {                                       // descending bucket starts: lane l owns buckets 63-2l, 62-2l
        const uint32_t c0 = s_cnt[63 - 2 * tid], c1 = s_cnt[62 - 2 * tid];
        uint32_t inc = c0 + c1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (tid >= o) inc += v; }
        s_cur[63 - 2 * tid] = inc - c0 - c1;
        s_cur[62 - 2 * tid] = inc - c1;
    }
    __syncthreads();
    for (int t = tid; t < T; t += 1024) {
        const uint2 r = ranges[t];
        order[atomicAdd(&s_cur[min(63u, (r.y - r.x) >> shift)], 1u)] = (uint32_t)t;
    }
}

// Empty tiles stay (0,0) like the reference's zero-initialised imgState.ranges.  prev: the previous view's header when
// several views share the binning buffer (this view's lists start where that view's end), else null.  tile_order null:
// the tile order is built later over all views (launch_tile_order).  With slabs == 0 (P == 0) every
// list is empty: ranges (0,0), R = 0, and the tile order of all-empty tiles.  count_host: the caller's page-locked
// host word for R, written straight from here (no copy in the stream between here and the scatter), or null.
// One CTA of 1024 threads (1-D or 32 x 32); slab_sum is read through L2 (other CTAs wrote it).
__device__ __forceinline__ void bin_starts_cta(int T, int slabs, uint32_t* __restrict__ slab_sum, uint2* ranges,
                                               GeomHeader* header, const GeomHeader* prev, long long capacity,
                                               uint32_t* __restrict__ tile_order, uint32_t* __restrict__ bwd_work,
                                               volatile int* count_host) {
    __shared__ uint32_t s_warp[32];
    const uint32_t base = prev ? __ldcg(&prev->list_base) + __ldcg(&prev->num_rendered) : 0u;
    const int tid = threadIdx.x + blockDim.x * threadIdx.y, lane = tid & 31, warp = tid >> 5;
    const int per = (T + 1023) / 1024;
    const int t0 = min(T, tid * per), t1 = min(T, t0 + per);
    uint32_t sum = 0;
    for (int t = t0; t < t1; ++t)
        for (int k = 0; k < slabs; ++k) sum += __ldcg(slab_sum + (size_t)k * T + t);
    uint32_t inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        const uint32_t wv = s_warp[lane];
        uint32_t wi = wv;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += v; }
        s_warp[lane] = wi - wv;
        if (lane == 31) {
            header->num_rendered = wi;
            header->list_base = base;
            if (count_host) *count_host = (int)wi;        // fenced after the ranges, by this thread
        }
    }
    __syncthreads();
    uint32_t run = base + s_warp[warp] + inc - sum;
    for (int t = t0; t < t1; ++t) {
        uint32_t n = 0;
        for (int k = 0; k < slabs; ++k) { const uint32_t v = __ldcg(slab_sum + (size_t)k * T + t); slab_sum[(size_t)k * T + t] = run + n; n += v; }
        // on overflow (R > capacity: the host grows the buffer and re-runs) keep every range inside the buffer
        ranges[t] = n ? make_uint2((uint32_t)min((long long)run, capacity), (uint32_t)min((long long)run + n, capacity))
                      : make_uint2(0u, 0u);
        run += n;
    }
    // R reaches the host before the kernel counts as complete (by now the store has mostly travelled)
    if (count_host && tid == 31) __threadfence_system();
    __syncthreads();                                      // every range written above is visible to the whole CTA
    if (tile_order) tile_order_cta(T, ranges, tile_order, bwd_work);
}

// Several views: the tile order of the tall grid, over the ranges every view's bin_starts wrote.
__global__ void __launch_bounds__(1024) tile_order_kernel(int T, const uint2* ranges, uint32_t* __restrict__ tile_order,
                                                          uint32_t* __restrict__ bwd_work) {
    tile_order_cta(T, ranges, tile_order, bwd_work);
}

// P == 0: every list empty (ranges (0,0), R = 0) and the tile order of all-empty tiles, by the same routine.
__global__ void __launch_bounds__(1024) bin_starts_kernel(int T, uint2* ranges, GeomHeader* header,
                                                          uint32_t* __restrict__ tile_order, uint32_t* __restrict__ bwd_work) {
    bin_starts_cta(T, 0, nullptr, ranges, header, nullptr, 0, tile_order, bwd_work, nullptr);
}

__global__ void __launch_bounds__(1024) bin_apply_kernel(int T, int chunks, uint32_t* __restrict__ M,
                                                         const uint32_t* __restrict__ slab_start) {
    __shared__ uint32_t s[32][33];
    const int tx = threadIdx.x, gy = threadIdx.y;
    const int t = blockIdx.x * 32 + tx;
    const int c0 = blockIdx.y * BIN_SLAB + gy * BIN_G;
    uint32_t v[BIN_G], sum = 0;
#pragma unroll
    for (int i = 0; i < BIN_G; ++i) {
        v[i] = (t < T && c0 + i < chunks) ? M[(size_t)(c0 + i) * T + t] : 0u;
        sum += v[i];
    }
    s[gy][tx] = sum;
    __syncthreads();
    if (gy == 0) {
        uint32_t acc = t < T ? slab_start[(size_t)blockIdx.y * T + t] : 0u;
#pragma unroll
        for (int g = 0; g < 32; ++g) { const uint32_t x = s[g][tx]; s[g][tx] = acc; acc += x; }
    }
    __syncthreads();
    uint32_t run = s[gy][tx];
    if (t < T) {
#pragma unroll
        for (int i = 0; i < BIN_G; ++i) {
            if (c0 + i < chunks) M[(size_t)(c0 + i) * T + t] = run;
            run += v[i];
        }
        if (c0 < chunks && chunks <= c0 + BIN_G) M[(size_t)chunks * T + t] = run;   // the group holding the last chunk
    }
}

// Debug only (r3dg_raster_debug_copy id 10): the reference's sorted 64-bit keys, rebuilt from the
// lists: (tile << 32) | depth bits of the listed Gaussian.
__global__ void rebuild_keys_kernel(int T, const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                                    const float* __restrict__ rec, int recf, long long limit, uint64_t* __restrict__ keys) {
    for (int t = blockIdx.x; t < T; t += gridDim.x) {
        const uint2 r = ranges[t];
        for (long long i = (long long)r.x + threadIdx.x; i < (long long)r.y && i < limit; i += blockDim.x)
            keys[i] = ((uint64_t)(uint32_t)t << 32) | (uint64_t)__float_as_uint(rec[(size_t)point_list[i] * recf + 6]);
    }
}

int launch_rebuild_keys(int T, const void* ranges, const uint32_t* point_list, const float* rec, int recf,
                        long long limit, uint64_t* keys, cudaStream_t stream) {
    rebuild_keys_kernel<<<1024, 128, 0, stream>>>(T, (const uint2*)ranges, point_list, rec, recf, limit, keys);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

// shared memory of bin_scatter: the per-tile array, the per-warp bitmaps, the per-position ids and block
// rectangles + a staging area of up to 12 entries per Gaussian, as far as it fits (>= CH entries, since one tile
// can receive every Gaussian of the chunk); a copy of the chunk's first slots per tile where that still leaves the
// full staging area (up to 1080p tile counts), otherwise step 3 reads them from M.  A larger staging area is
// slower at the headline: it spares the few heaviest chunks a second window but leaves less of the SM's
// L1 / shared-memory split to L1.
constexpr size_t kBinSmemMax = 220 * 1024;                // + ~5 KB static
static size_t bin_tile_bytes(int T) { return (((size_t)T + 3) & ~(size_t)3) * 4; }
static size_t bin_table_bytes(int T, int CH) {
    return bin_tile_bytes(T) + (size_t)(BIN_SCATTER_THREADS / 32) * 2 * ((CH + 31) / 32) * 4 + (size_t)CH * 12;
}

int check_binning_limits(const RasterBuffers& b) {
    const int CH = b.chunk_len;
    if (b.gx > 65535 || b.gy > 65535 || b.tiles > 65535 || CH > 65536 ||
        bin_table_bytes(b.tiles, CH) + (size_t)CH * 4 > kBinSmemMax) return R3DG_ERR_UNSUPPORTED;
    return 0;
}

int launch_binning(int P, const RasterBuffers& b, int num_sms, cudaStream_t stream, stage_mark_fn mark,
                   int* num_rendered_host, void* count_ready_event) {
    const int gx = b.gx, T = b.tiles, CH = b.chunk_len, chunks = b.chunks;
    if (int rc = check_binning_limits(b)) return rc;
    const size_t smem_max = kBinSmemMax;
    const size_t tile_bytes = bin_tile_bytes(T);
    size_t tbl_bytes = bin_table_bytes(T, CH);
    const size_t full_stage = std::min<size_t>((size_t)CH * 12, (size_t)BIN_MAX_LONG * BIN_LONG_RUN);
    const int starts_in_smem = tbl_bytes + tile_bytes + full_stage * 4 <= smem_max ? 1 : 0;
    if (starts_in_smem) tbl_bytes += tile_bytes;
    int cap = (int)std::min<size_t>((smem_max - tbl_bytes) / 4, full_stage);
    if (const char* e = getenv("R3DG_BIN_STAGE_CAP")) cap = std::max(CH, std::min(cap, atoi(e)));   // tests: force the multi-window path
    int rc = launch_sort(b.header, b.sort, b.sort_layout, P, num_sms, stream);
    if (rc != 0) return rc;
    mark(2, stream);
    const size_t smem_count = (size_t)T * 4;
    const size_t smem_scatter = tbl_bytes + (size_t)cap * 4;
    R3DG_CUDA_TRY(allow_dyn_smem<bin_count_kernel>(smem_count));
    R3DG_CUDA_TRY(allow_dyn_smem<bin_scatter_kernel>(smem_scatter));
    const uint32_t* va = (const uint32_t*)(b.sort + b.sort_layout.vals_a);
    const uint32_t* vb = (const uint32_t*)(b.sort + b.sort_layout.vals_b);
    uint32_t* M = b.bin_matrix;
    const int slabs = (chunks + BIN_SLAB - 1) / BIN_SLAB;
    const dim3 sgrid((T + 31) / 32, slabs), sblock(32, 32);
    bin_count_kernel<<<chunks, BIN_COUNT_THREADS, smem_count, stream>>>(P, T, gx, CH, b.header, va, vb, b.rects, M);
    mark(3, stream);
    // the instance count exists after bin_starts: hand it to the host early (the scatter and the compositor are still
    // to run).  Page-locked host memory is mapped into the device's address space: bin_starts stores the count there
    // itself, which spares the stream a device-to-host copy between two kernels.  Pageable memory takes the copy.
    int* count_host = nullptr;
    if (num_rendered_host) {
        cudaPointerAttributes pa;
        if (cudaPointerGetAttributes(&pa, num_rendered_host) == cudaSuccess && pa.type == cudaMemoryTypeHost &&
            pa.devicePointer && pa.hostPointer)
            count_host = (int*)((char*)pa.devicePointer + ((char*)num_rendered_host - (char*)pa.hostPointer));
        else
            cudaGetLastError();                           // clear the query's error state
    }
    bin_colsum_kernel<<<sgrid, sblock, 0, stream>>>(T, chunks, slabs, M, b.slab_sum, b.ranges, b.header, b.prev_header,
                                                    b.capacity, b.tile_order, b.bwd_work, count_host);
    if (num_rendered_host && !count_host)
        R3DG_CUDA_TRY(cudaMemcpyAsync(num_rendered_host, b.header, sizeof(int), cudaMemcpyDeviceToHost, stream));
    if (count_ready_event) R3DG_CUDA_TRY(cudaEventRecord((cudaEvent_t)count_ready_event, stream));
    bin_apply_kernel<<<sgrid, sblock, 0, stream>>>(T, chunks, M, b.slab_sum);
    mark(4, stream);
    bin_scatter_kernel<<<chunks, BIN_SCATTER_THREADS, smem_scatter, stream>>>(
        P, T, gx, (1ull << 32) / (unsigned long long)gx + 1ull, CH, cap, b.header, va, vb, b.rects, b.brects, M, b.point_list,
        b.bmask, b.cmask, b.capacity, starts_in_smem, b.row_base);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_empty_binning(const RasterBuffers& b, cudaStream_t stream) {
    bin_starts_kernel<<<1, 1024, 0, stream>>>(b.V * b.tiles, b.ranges, b.header, b.tile_order, b.bwd_work);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_tile_order(const RasterBuffers& b, cudaStream_t stream) {
    tile_order_kernel<<<1, 1024, 0, stream>>>(b.V * b.tiles, b.ranges, b.tile_order, b.bwd_work);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
