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
//   bin_colsum/starts/apply    : exclusive scan of every column of M (per tile over the chunks),
//                                exclusive scan of the tile totals -> ranges[tile], R; M becomes the
//                                absolute first slot of (chunk, tile);
//   bin_scatter                : every chunk re-walks its Gaussians and writes each instance to
//                                M[chunk][tile] + (rank inside the chunk, in sequence order).
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
__global__ void __launch_bounds__(256) bin_count_kernel(int P, int T, int gx, int CH,
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
//   1. recount the chunk per tile (as bin_count), exclusive scan -> local CSR offsets;
//   2. unordered append: one thread per Gaussian, slot = shared atomicAdd on the tile's cursor,
//      entry = {Gaussian id, tile << 16 | position in the chunk};
//   3. one thread per staged entry: rank = number of entries of its run (same tile) that come
//      earlier in the sequence; global slot = M[chunk][tile] + rank.  A warp's lanes hold
//      consecutive staged entries, i.e. whole runs, whose global slots are contiguous: the
//      stores coalesce into a few sectors per run instead of one transaction per entry.
// A chunk whose instances exceed the staging area is handled in several windows of tiles.
#define BIN_SCATTER_THREADS 1024
#define BIN_LONG_RUN 24            // runs longer than this are ranked through the bitmap
#define BIN_MAX_LONG 2048          // >= staging capacity / BIN_LONG_RUN

__global__ void __launch_bounds__(BIN_SCATTER_THREADS) bin_scatter_kernel(
    int P, int T, int gx, int CH, int cap, const GeomHeader* __restrict__ header, const uint32_t* __restrict__ vals_a,
    const uint32_t* __restrict__ vals_b, const uint2* __restrict__ rects, const uint32_t* __restrict__ M,
    uint32_t* __restrict__ point_list, long long capacity) {
    extern __shared__ __align__(16) uint32_t bin_smem[];
    uint32_t* a = bin_smem;                               // [T] counts -> exclusive offsets -> cursors
    const int words = (CH + 31) >> 5;                     // bitmap over the chunk positions, per warp
    uint32_t* bitmaps = bin_smem + (((size_t)T + 3) & ~(size_t)3);
    uint2* stage = reinterpret_cast<uint2*>(bitmaps + (size_t)(BIN_SCATTER_THREADS / 32) * 2 * words);
    __shared__ uint32_t s_warp[BIN_SCATTER_THREADS / 32];
    __shared__ int s_hi;
    __shared__ uint32_t s_total, s_nlong;
    __shared__ uint16_t s_long[BIN_MAX_LONG];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t* __restrict__ order = (header->sort_exec & 1u) ? vals_b : vals_a;
    const int c = blockIdx.x;
    const int j0 = c * CH, j1 = min(P, j0 + CH);
    const uint32_t* __restrict__ row = M + (size_t)c * T;
    for (int t = tid; t < T; t += BIN_SCATTER_THREADS) a[t] = 0u;
    __syncthreads();
    // ---- 1. per-tile counts of the chunk, exclusive scan over the tiles --------------------------
    for (int j = j0 + tid; j < j1; j += BIN_SCATTER_THREADS) {
        const uint2 r = rects[order[j]];
        const uint32_t w = r.y & 0xffffu, h = r.y >> 16;
        // one flat loop over the w*h tiles (lanes have different rectangles: nested loops would
        // serialise max(h) * max(w) trips per warp instead of max(w*h))
        uint32_t tile = (r.x >> 16) * (uint32_t)gx + (r.x & 0xffffu), x = 0;
        const uint32_t n = w * h, skip = (uint32_t)gx - w;
#pragma unroll 1
        for (uint32_t k = 0; k < n; ++k) {
            atomicAdd(&a[tile], 1u);
            ++tile;
            if (++x == w) { x = 0; tile += skip; }
        }
    }
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
            const uint32_t g = order[j];
            const uint2 r = rects[g];
            const uint32_t w = r.y & 0xffffu, h = r.y >> 16;
            uint32_t tile = (r.x >> 16) * (uint32_t)gx + (r.x & 0xffffu), x = 0;
            const uint32_t n = w * h, skip = (uint32_t)gx - w;
            const uint32_t seq = (uint32_t)(j - j0);
#pragma unroll 1
            for (uint32_t k = 0; k < n; ++k) {
                if ((int)tile >= lo && (int)tile < hi) {
                    const uint32_t slot = atomicAdd(&a[tile], 1u) - first;
                    stage[slot] = make_uint2(g, (tile << 16) | seq);
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
            const uint2 e = stage[i];
            const int t = (int)(e.y >> 16);
            const uint32_t seq = e.y & 0xffffu;
            const uint32_t rb = (t > lo ? a[t - 1] : first) - first, re = a[t] - first;
            if (re - rb > BIN_LONG_RUN) continue;
            uint32_t rank = 0;
#pragma unroll 2
            for (uint32_t k = rb; k < re; ++k) rank += ((stage[k].y & 0xffffu) < seq) ? 1u : 0u;
            const long long pos = (long long)row[t] + rank;
            if (pos < capacity) point_list[pos] = e.x;
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
                for (uint32_t k = rb + lane; k < re; k += 32) { const uint32_t sq = stage[k].y & 0xffffu; atomicOr(&bm[sq >> 5], 1u << (sq & 31u)); }
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
                const uint32_t base = row[t];
#pragma unroll 1
                for (uint32_t k = rb + lane; k < re; k += 32) {
                    const uint2 e = stage[k];
                    const uint32_t sq = e.y & 0xffffu;
                    const uint32_t rank = bp[sq >> 5] + (uint32_t)__popc(bm[sq >> 5] & ((1u << (sq & 31u)) - 1u));
                    const long long pos = (long long)base + rank;
                    if (pos < capacity) point_list[pos] = e.x;
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
//   bin_colsum  : slab_sum[slab][tile] = sum of the slab's rows;
//   bin_starts  : one CTA; exclusive scan of the tile totals -> ranges, R; per slab and tile the
//                 absolute first slot (tile start + earlier slabs) -> slab_sum in place;
//   bin_apply   : every thread keeps its BIN_G counts in registers, the CTA scans the 32 group sums
//                 through shared memory and M is rewritten as ABSOLUTE first slots.
#define BIN_G 16
#define BIN_SLAB (32 * BIN_G)

__global__ void __launch_bounds__(1024) bin_colsum_kernel(int T, int chunks, const uint32_t* __restrict__ M,
                                                          uint32_t* __restrict__ slab_sum) {
    __shared__ uint32_t s[32][33];
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
}

// Empty tiles stay (0,0) like the reference's zero-initialised imgState.ranges.
__global__ void __launch_bounds__(1024) bin_starts_kernel(int T, int slabs, uint32_t* __restrict__ slab_sum,
                                                          uint2* __restrict__ ranges, GeomHeader* header,
                                                          long long capacity) {
    __shared__ uint32_t s_warp[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per = (T + 1023) / 1024;
    const int t0 = min(T, tid * per), t1 = min(T, t0 + per);
    uint32_t sum = 0;
    for (int t = t0; t < t1; ++t)
        for (int k = 0; k < slabs; ++k) sum += slab_sum[(size_t)k * T + t];
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
        if (lane == 31) header->num_rendered = wi;
    }
    __syncthreads();
    uint32_t run = s_warp[warp] + inc - sum;
    for (int t = t0; t < t1; ++t) {
        uint32_t n = 0;
        for (int k = 0; k < slabs; ++k) { const uint32_t v = slab_sum[(size_t)k * T + t]; slab_sum[(size_t)k * T + t] = run + n; n += v; }
        // on overflow (R > capacity: the host grows the buffer and re-runs) keep every range inside the buffer
        ranges[t] = n ? make_uint2((uint32_t)min((long long)run, capacity), (uint32_t)min((long long)run + n, capacity))
                      : make_uint2(0u, 0u);
        run += n;
    }
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

int launch_binning(int P, int W, int H, char* geom, const GeomLayout& gl, char* img, const ImgLayout& il,
                   char* bin, const BinLayout& bl, int num_sms, cudaStream_t stream, stage_mark_fn mark,
                   int* num_rendered_host, void* count_ready_event) {
    const int gx = (W + R3DG_TILE - 1) / R3DG_TILE, gy = (H + R3DG_TILE - 1) / R3DG_TILE;
    const int T = gx * gy;
    const int CH = bin_chunk_len(P, (size_t)T);
    const int chunks = (P + CH - 1) / CH;
    // shared memory of bin_scatter: the per-tile array + as large a staging area as fits (>= CH entries,
    // since one tile can receive every Gaussian of the chunk)
    const size_t smem_max = 220 * 1024;                   // + ~5 KB static
    const size_t tbl_bytes = (((size_t)T + 3) & ~(size_t)3) * 4 +
                             (size_t)(BIN_SCATTER_THREADS / 32) * 2 * ((CH + 31) / 32) * 4;      // per-tile array + per-warp bitmaps
    if (gx > 65535 || gy > 65535 || T > 65535 || tbl_bytes + (size_t)CH * 8 > smem_max) return R3DG_ERR_UNSUPPORTED;
    int cap = (int)std::min<size_t>(std::min<size_t>((smem_max - tbl_bytes) / 8, (size_t)CH * 12), (size_t)BIN_MAX_LONG * BIN_LONG_RUN);
    if (const char* e = getenv("R3DG_BIN_STAGE_CAP")) cap = std::max(CH, std::min(cap, atoi(e)));   // tests: force the multi-window path
    GeomHeader* header = (GeomHeader*)(geom + gl.header);
    const SortLayout sl(P);
    char* sbuf = geom + gl.sort;
    int rc = launch_sort(header, sbuf, sl, P, num_sms, stream);
    if (rc != 0) return rc;
    mark(2, stream);
    const size_t smem_count = (size_t)T * 4;
    const size_t smem_scatter = tbl_bytes + (size_t)cap * 8;
    static size_t attr_smem[2] = {0, 0};
    if (smem_count > attr_smem[0]) {
        R3DG_CUDA_TRY(cudaFuncSetAttribute(bin_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_count));
        attr_smem[0] = smem_count;
    }
    if (smem_scatter > attr_smem[1]) {
        R3DG_CUDA_TRY(cudaFuncSetAttribute(bin_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_scatter));
        attr_smem[1] = smem_scatter;
    }
    const uint32_t* va = (const uint32_t*)(sbuf + sl.vals_a);
    const uint32_t* vb = (const uint32_t*)(sbuf + sl.vals_b);
    const uint2* rects = (const uint2*)(geom + gl.rects);
    uint32_t* M = (uint32_t*)(img + il.bin_matrix);
    uint2* ranges = (uint2*)(img + il.ranges);
    uint32_t* slab_sum = (uint32_t*)(img + il.slab_sum);
    uint32_t* point_list = (uint32_t*)(bin + bl.point_list);
    const int slabs = (chunks + BIN_SLAB - 1) / BIN_SLAB;
    const dim3 sgrid((T + 31) / 32, slabs), sblock(32, 32);
    bin_count_kernel<<<chunks, 256, smem_count, stream>>>(P, T, gx, CH, header, va, vb, rects, M);
    mark(3, stream);
    bin_colsum_kernel<<<sgrid, sblock, 0, stream>>>(T, chunks, M, slab_sum);
    bin_starts_kernel<<<1, 1024, 0, stream>>>(T, slabs, slab_sum, ranges, header, bl.capacity);
    // the instance count exists now: hand it to the host early (the scatter and the compositor are still to run)
    if (num_rendered_host) R3DG_CUDA_TRY(cudaMemcpyAsync(num_rendered_host, header, sizeof(int), cudaMemcpyDeviceToHost, stream));
    if (count_ready_event) R3DG_CUDA_TRY(cudaEventRecord((cudaEvent_t)count_ready_event, stream));
    bin_apply_kernel<<<sgrid, sblock, 0, stream>>>(T, chunks, M, slab_sum);
    mark(4, stream);
    bin_scatter_kernel<<<chunks, BIN_SCATTER_THREADS, smem_scatter, stream>>>(P, T, gx, CH, cap, header, va, vb, rects, M,
                                                                               point_list, bl.capacity);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
