// Shared device-side definitions: the packed per-Gaussian record, the radix-sort layout and
// small helpers.  Nothing here is visible through the C ABI (include/r3dg_b200.h); the layout
// of the rasterizer's work buffers belongs to api.cu.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>

#define R3DG_TILE 16                 // 16x16 pixel tiles (reference config.h:15-17, fixed by parity)
#define R3DG_MAX_S_FWD 33            // forward.cu:312  F[33]
#define R3DG_MAX_S_BWD 24            // backward.cu:449 collected_features[24 * BLOCK_SIZE]

namespace r3dg {

// ---------------------------------------------------------------------------------------------
// Packed per-Gaussian record written by the projection kernel and gathered by the compositors.
// One 16-byte-aligned AoS row of RECF = 8 + 4*NG floats per Gaussian:
//   [0] mean2D.x [1] mean2D.y [2] conic.a [3] conic.b | [4] conic.c [5] opacity [6] depth(view z)
//   [7] radius (int bits) | [8..] channels = {r,g,b,f0..f(S-1)} zero-padded to 4*NG
// A compositor instance touches exactly this one row (2 sectors for S=5), instead of the
// reference's 5 separate arrays (means2D, conic_opacity, depths, colors, features).
// Ray-depth mode (r3dg_raster_fwd_args.ray_depth) appends one group: [8 + 4*NG] depth plane p.x [+1] p.y [+2, +3] 0.
// ---------------------------------------------------------------------------------------------
__host__ __device__ inline int num_groups(int S) { return (3 + S + 3) / 4; }
__host__ __device__ inline int rec_floats(int S) { return 8 + 4 * num_groups(S); }
__host__ __device__ inline int rec_floats(int S, bool ray_depth) { return rec_floats(S) + (ray_depth ? 4 : 0); }

// Per-Gaussian gradient row accumulated by the backward compositor, same width as the record:
//   [0] dmean2D.x [1] dmean2D.y [2] dmean2D.z(depth) [3] dopacity | [4] dconic.a [5] dconic.b
//   [6] dconic.c  [7] unused | [8..] d channels (ray-depth mode: then dL/dp.x, dL/dp.y, 0, 0)
// A warp reduces the row across its 32 pixels and adds it with one vector of atomics.

struct GeomHeader {               // first 256 bytes of the geometry buffer
    uint32_t num_rendered;        // R = total (tile, Gaussian) instances (may exceed capacity)
    uint32_t scan_ticket;         // dynamic block id for the chained scan (debug point_offsets only)
    uint32_t sort_ticket[8];      // dynamic tile id per radix pass
    uint32_t depth_or;            // OR of the sort keys (visible depth bit patterns)
    uint32_t depth_nor;           // OR of their complements: bit varies across keys iff set in both
    uint32_t sort_exec;           // number of radix passes actually executed (parity = result buffer)
    uint32_t bin_ticket;          // CTAs of bin_colsum done (the last one scans the tile totals)
    uint32_t list_base;           // first binning slot of this view's lists (several views share one binning buffer)
    uint32_t pad[49];
};
static_assert(sizeof(GeomHeader) == 256, "header size");

inline __host__ __device__ size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

#define R3DG_SCAN_ITEMS 2048       // items per chained-scan block

// ---- radix sort of (u32 key, u32 value) pairs (radix_sort.cu) ---------------------------------
#define R3DG_SORT_THREADS 256
#define R3DG_SORT_ITEMS 8
#define R3DG_SORT_TILE (R3DG_SORT_THREADS * R3DG_SORT_ITEMS)   // 2048 pairs per onesweep tile
#define R3DG_SORT_MAX_PASSES 4

struct SortLayout {
    size_t keys_a, keys_b, vals_a, vals_b, hist, tilecnt, total;
    long long n, tiles, plane_words;
    __host__ __device__ SortLayout(long long n_) : n(n_) {
        tiles = (n_ + R3DG_SORT_TILE - 1) / R3DG_SORT_TILE + 1;
        plane_words = tiles * 256;                          // digit counts per tile; two planes, used alternately
        size_t off = 0;
        keys_a = off; off = align_up(off + (size_t)n_ * 4, 256);
        keys_b = off; off = align_up(off + (size_t)n_ * 4, 256);
        vals_a = off; off = align_up(off + (size_t)n_ * 4, 256);
        vals_b = off; off = align_up(off + (size_t)n_ * 4, 256);
        hist = off;   off = align_up(off + (size_t)R3DG_SORT_MAX_PASSES * 256 * 4, 256);
        tilecnt = off;
        off = align_up(off + (size_t)2 * plane_words * 4, 256);
        total = off;
    }
};

// The key bits above the highest VARYING bit are identical in every key and need no pass; the
// remaining nb bits are split evenly over ceil(nb/8) passes of w <= 8 bits.  All of it is decided
// on the device from (key_or & key_nor); the k-th pass reads buffer (k & 1), so the result lives
// in buffer (sort_exec & 1).
__device__ __forceinline__ void sort_plan(uint32_t diff, int& passes, int& w) {
    const int nb = 32 - __clz(diff);                      // __clz(0) == 32
    passes = (nb + 7) >> 3;
    w = passes ? (nb + passes - 1) / passes : 0;
}

// ---- depth-ordered tile binning (binning.cu) -------------------------------------------------
// The depth-sorted Gaussians are cut into `chunks` runs of CH; M[chunk][tile] first counts the
// instances a chunk adds to a tile, then (scanned down the columns) is the chunk's first slot
// inside the tile's list, and row M[chunks] holds the (unclamped) end of every list.
#define R3DG_BIN_MAX_CHUNKS 1024
inline int bin_max_chunks(size_t T) {                                 // the most chunks M holds for T tiles
    if (const char* e = getenv("R3DG_BIN_MAX_CHUNKS")) { const int v = atoi(e); if (v >= 1 && v <= R3DG_BIN_MAX_CHUNKS) return v; }   // tests: long chunks
    size_t c = ((size_t)1 << 26) / (T ? T : 1);
    return (int)(c < 296 ? 296 : (c > R3DG_BIN_MAX_CHUNKS ? R3DG_BIN_MAX_CHUNKS : c));
}
inline int bin_chunk_len(int P, int max_chunks) {                     // Gaussians per chunk, multiple of 256
    // ~3 chunks per SM for load balance, 512..2048 Gaussians (longer per-tile runs coalesce better,
    // the staging area of bin_scatter bounds it), and never more chunks than M has rows
    int ch = ((P + 443) / 444 + 255) / 256 * 256;
    ch = ch < 512 ? 512 : (ch > 2048 ? 2048 : ch);
    const int need = ((P + max_chunks - 1) / max_chunks + 255) / 256 * 256;
    return ch > need ? ch : need;
}

// Relaxed GPU-scope accesses for the look-back descriptors (flag and value share one word, so no
// further ordering is needed); `volatile` asm so that polling loops really re-load.
// ---- asynchronous global -> shared copies (LDGSTS): no register staging, overlap with math -----
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// ---- TMA-unit bulk copies (cp.async.bulk, SASS UBLKCP) completing on an mbarrier (SYNCS) -------------------
// One instruction moves a contiguous, 16-byte aligned slab global -> shared with no register staging and no
// per-thread address arithmetic; completion is signalled by transaction bytes on a shared-memory mbarrier.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// shared -> global bulk store (UBLKCP.G.S): the issuing thread commits and waits until the source may be reused
__device__ __forceinline__ void bulk_copy_s2g(void* gmem_dst, const void* smem_src, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;\n" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// Asynchronous, coalesced copy of a CTA's [nvalid][rowf] float slab into the TRANSPOSED shared slab
// s[k * ld + t] (element k of row t): every warp instruction moves 32 consecutive floats (128 B of
// global memory) to 32 different banks.  nthreads = blockDim.x.  rows: null, or a bit mask of the rows to copy (bit
// t & 31 of rows[t >> 5]); the other rows' slab entries are left as they are.
__device__ __forceinline__ void load_rows_transposed_async(float* s, int ld, const float* __restrict__ src,
                                                           int nvalid, int rowf, int nthreads,
                                                           const uint32_t* rows = nullptr) {
    const int total = nvalid * rowf;
    const int dq = nthreads / rowf, dm = nthreads - dq * rowf;
    int t = (int)threadIdx.x / rowf, k = (int)threadIdx.x - t * rowf;
    for (int i = threadIdx.x; i < total; i += nthreads) {
        if (!rows || ((rows[t >> 5] >> (t & 31)) & 1u)) cp_async4(s + k * ld + t, src + i);
        k += dm; t += dq;
        if (k >= rowf) { k -= rowf; ++t; }
    }
}

__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_gpu(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// --- exact-association arithmetic (see tools/sass_trace.py / DESIGN.md "bit-exact binning") ----
// Explicit intrinsics are never re-contracted by nvcc, so the association below is what runs.
__device__ __forceinline__ float fma_(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float mul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_(float a, float b) { return __fsub_rn(a, b); }
// c += w * x on the lanes where `on` holds, as predicated FFMAs: no branch and no select, and a lane that is off keeps
// its accumulators bit for bit even when x is not finite (what the reference's per-thread `continue` guarantees).
__device__ __forceinline__ void fma4_if(bool on, float w, const float4& x, float& c0, float& c1, float& c2, float& c3) {
    asm("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %4, 0;\n\t@q fma.rn.f32 %0, %5, %6, %0;\n\t@q fma.rn.f32 %1, %5, %7, %1;\n\t"
        "@q fma.rn.f32 %2, %5, %8, %2;\n\t@q fma.rn.f32 %3, %5, %9, %3;\n\t}"
        : "+f"(c0), "+f"(c1), "+f"(c2), "+f"(c3)
        : "r"((unsigned)on), "f"(w), "f"(x.x), "f"(x.y), "f"(x.z), "f"(x.w));
}
__device__ __forceinline__ void fma_add_if(bool on, float w, float x, float& c, float& sum) {   // c += w * x ; sum += w
    asm("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %2, 0;\n\t@q fma.rn.f32 %0, %3, %4, %0;\n\t@q add.rn.f32 %1, %1, %3;\n\t}"
        : "+f"(c), "+f"(sum) : "r"((unsigned)on), "f"(w), "f"(x));
}
__device__ __forceinline__ float div_(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float rcp_(float a) { return __frcp_rn(a); }
__device__ __forceinline__ float sqrt_(float a) { return __fsqrt_rn(a); }
// a0*b0 + a1*b1 + a2*b2 with the middle product as the plain multiply (reference SASS pattern)
__device__ __forceinline__ float dot3_(float a0, float b0, float a1, float b1, float a2, float b2) {
    return fma_(a2, b2, fma_(a0, b0, mul_(a1, b1)));
}
__device__ __forceinline__ float xform_row_(const float* __restrict__ m, int r, float x, float y, float z) {
    return add_(dot3_(x, m[r], y, m[4 + r], z, m[8 + r]), m[12 + r]);
}

// Mip-Splatting's 3D filter of size f on scales s (filter3d.py fold, in the same op order): s'_k = sqrt(s_k^2 + f^2)
// replaces s in place, and the opacity factor coef = sqrt((r_0 r_1) r_2), r_k = s_k^2 / s'_k^2 (1 when s'_k = 0), is
// returned.  The per-axis ratios do not underflow where det(Sigma) would (s ~ 1e-7).  f = 0: s' = |s|, coef = 1 (for
// s = 0 and every s whose square is a normal float).
__device__ __forceinline__ float filter3d_fold(float (&s)[3], float f) {
    const float g = mul_(f, f);
    float r[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float q = mul_(s[k], s[k]), e = add_(q, g);
        s[k] = sqrt_(e);
        r[k] = e == 0.0f ? 1.0f : div_(q, e);
    }
    return sqrt_(mul_(mul_(r[0], r[1]), r[2]));
}

// getRect (reference auxiliary.h:46-56), /16 compiled to an exact *0.0625f
__device__ __forceinline__ void get_rect(float px, float py, int radius, int gx, int gy, int& x0,
                                         int& y0, int& x1, int& y1) {
    const float r = (float)radius;
    x0 = min(gx, max(0, (int)mul_(sub_(px, r), 0.0625f)));
    y0 = min(gy, max(0, (int)mul_(sub_(py, r), 0.0625f)));
    x1 = min(gx, max(0, (int)mul_(add_(add_(add_(px, r), 16.0f), -1.0f), 0.0625f)));
    y1 = min(gy, max(0, (int)mul_(add_(add_(add_(py, r), 16.0f), -1.0f), 0.0625f)));
}

// ---------------------------------------------------------------------------------------------
// Conservative sub-tile culling.  A tile's 16x16 pixels are owned by 8 warps, each a compact 8x4
// pixel block.  touch_block() returns false only if NO pixel of the block whose first pixel is
// (X0, Y0) can pass the reference's per-pair tests (power <= 0 and alpha >= 1/255,
// forward.cu:345-354) for this Gaussian:  alpha >= 1/255  =>  q(d) = a dx^2 + 2b dx dy + c dy^2
// <= tau = 2 ln(255 o).  The minimum of the convex quadratic over the block's (continuous)
// rectangle is found on its four edges; a slack of 1 + 1e-5 * |largest term| (>> fp32 rounding of
// either evaluation) keeps the test conservative, so skipped pairs are exactly pairs the
// reference's arithmetic would have rejected and per-pixel results stay bit-identical.
// Non-positive-definite or NaN conics are never culled.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool touch_block(const float4 A, const float4 B, float X0, float Y0) {
    const float gx = A.x, gy = A.y, ca = A.z, cb = A.w, cc = B.x, op = B.y;
    if (op < 1.0f / 255.0f) return false;                    // alpha <= op < 1/255 everywhere
    if (!(ca > 0.0f && cc > 0.0f && ca * cc - cb * cb > 0.0f)) return true;
    const float tau = 2.0f * __logf(255.0f * op) ;
    if (!(tau >= 0.0f)) return true;                          // NaN opacity etc.
    const float u0 = gx - (X0 + 7.0f), u1 = gx - X0, v0 = gy - (Y0 + 3.0f), v1 = gy - Y0;
    if (u0 <= 0.0f && u1 >= 0.0f && v0 <= 0.0f && v1 >= 0.0f) return true;   // centre inside the block
    const float rc = __fdividef(-cb, cc), ra = __fdividef(-cb, ca);
    auto edge_u = [&](float U) {
        const float v = fminf(fmaxf(rc * U, v0), v1);
        return ca * U * U + 2.0f * cb * U * v + cc * v * v;
    };
    auto edge_v = [&](float V) {
        const float u = fminf(fmaxf(ra * V, u0), u1);
        return ca * u * u + 2.0f * cb * u * V + cc * V * V;
    };
    const float qmin = fminf(fminf(edge_u(u0), edge_u(u1)), fminf(edge_v(v0), edge_v(v1)));
    const float um = fmaxf(fabsf(u0), fabsf(u1)), vm = fmaxf(fabsf(v0), fabsf(v1));
    // slack also absorbs the approximate log/divide above (relative error ~1e-6 of tau <= ~12)
    const float slack = 1.0f + 1e-5f * (ca * um * um + cc * vm * vm + 2.0f * fabsf(cb) * um * vm);
    return !(qmin > tau + slack);
}

// ---------------------------------------------------------------------------------------------
// Conservative footprint of a Gaussian in units of the compositors' pixel blocks (8 px wide, 4 px high): the
// axis-aligned bounding box of the ellipse {q <= tau_b} around the projected centre, where every pixel that can pass
// the reference's alpha >= 1/255 test (q <= tau = 2 ln(255 o), evaluated in fp32) lies.  tau_b = 1.02 tau + 0.25
// absorbs the fp32 evaluation error of the per-pixel quadratic for conics with trace^2/det <= 6000 (error <=
// 2.4e-7 * 1.5 * trace^2/det * q); worse-conditioned, non-positive-definite or NaN conics get the full range.
// Packed {bx0 | bx1 << 16, by0 | by1 << 16}, inclusive block column / row indices; empty (bx0 > bx1) when the
// opacity is below 1/255.  This is only a PRE-filter (block_mask_of_rect, written by bin_scatter): the compositor
// still applies the exact ellipse / rectangle test to what passes, and the exact per-pixel tests to what passes that.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint2 block_rect(float gx, float gy, float ca, float cb, float cc, float op) {
    if (op < 1.0f / 255.0f) return make_uint2(1u, 0u);                       // bx0 = 1 > bx1 = 0: touches nothing
    const float det = ca * cc - cb * cb, tr = ca + cc;
    const float tau = 2.0f * __logf(255.0f * op);
    if (!(ca > 0.0f && cc > 0.0f && det > 0.0f && tr * tr <= 6000.0f * det && tau >= 0.0f)) return make_uint2(0xffff0000u, 0xffff0000u);
    const float tb = 1.02f * tau + 0.25f;
    const float hx = sqrtf(tb * cc / det) * 1.0001f + 0.01f, hy = sqrtf(tb * ca / det) * 1.0001f + 0.01f;
    auto blk = [](float v, float inv) { return (uint32_t)fminf(fmaxf(floorf(v * inv), 0.0f), 65535.0f); };
    // a box entirely left of / above the image maps to an empty range (pixels have coordinates >= 0)
    if (gx + hx < 0.0f || gy + hy < 0.0f) return make_uint2(1u, 0u);
    return make_uint2(blk(gx - hx, 0.125f) | (blk(gx + hx, 0.125f) << 16), blk(gy - hy, 0.25f) | (blk(gy + hy, 0.25f) << 16));
}

// The 8-bit block pre-filter mask of one (tile, Gaussian) instance: bit b = block b of the tile intersects the
// Gaussian's block rectangle.  c0 / r0 = first block column / row of the tile.
__device__ __forceinline__ uint32_t block_mask_of_rect(uint2 br, uint32_t c0, uint32_t r0) {
    const uint32_t bx0 = br.x & 0xffffu, bx1 = br.x >> 16, by0 = br.y & 0xffffu, by1 = br.y >> 16;
    // block rows r0 + [rlo, rhi] and columns c0 + [clo, chi] lie inside the rectangle: contiguous bit runs
    const int rlo = max((int)by0 - (int)r0, 0), rhi = min((int)by1 - (int)r0, 3);
    const int clo = max((int)bx0 - (int)c0, 0), chi = min((int)bx1 - (int)c0, 1);
    const uint32_t rows = rlo <= rhi ? (2u << rhi) - (1u << rlo) : 0u;
    const uint32_t cols = clo <= chi ? (2u << chi) - (1u << clo) : 0u;
    // block b = (row b >> 1, column b & 1): spread the row bits to even positions; times cols (0..3) places them in
    // column 0, column 1 or both (the spread bits are two apart, so the product has no carries)
    uint32_t spread = (rows | (rows << 2)) & 0x33u;
    spread = (spread | (spread << 1)) & 0x55u;
    return spread * cols;
}

// ---- warp-level stream compaction over per-instance mask bytes (compositors) ---------------------
// A warp walks its tile's mask bytes 128 entries at a time (one 4-byte word per lane), keeps the entries whose bit
// `bit` is set and appends their list positions, in list order, to a small circular queue in shared memory.  The
// lane-level ranks come from one warp scan of the per-lane popcounts.
#define R3DG_QCAP 256                      // queue slots per warp (>= 31 + 128 pending entries), power of two

__device__ __forceinline__ uint32_t warp_excl_scan(uint32_t v, int lane, uint32_t& total) {
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    total = __shfl_sync(0xffffffffu, inc, 31);
    return inc - v;
}

}  // namespace r3dg

#define R3DG_CUDA_TRY(expr)                                  \
    do {                                                     \
        cudaError_t _e = (expr);                             \
        if (_e != cudaSuccess) return -(int)_e;              \
    } while (0)
