// Stage 1 of the hot path: per-Gaussian projection / cull / covariance (reference K1,
// forward.cu:156-258), tile-count prefix sum (K2, rasterizer_impl.cu:287), key duplication
// (K4, rasterizer_impl.cu:70-111), tile ranges (K6, rasterizer_impl.cu:116-138) and
// markVisible (K13).  The radix sort (K5) lives in radix_sort.cu.
//
// Design notes
//  * one packed 16B-aligned record per Gaussian (common.cuh) is produced here so the compositors
//    gather one row instead of five arrays;
//  * the floating-point association of everything that feeds radii / tile rectangles / depth keys
//    is pinned with explicit round-to-nearest intrinsics to the association of the reference's
//    compiled binary, which makes point_list / ranges / n_contrib bit-identical;
//  * the instance count R never travels to the host inside the pipeline: kernels read it from
//    the geometry header, grids are sized from the SM count, and the binning buffer is
//    capacity-checked on the device.
#include <cstdio>
#include "common.cuh"
#include "kernels.h"
#include "sh.cuh"

namespace r3dg {

// computeCov3D, association pinned (see oracle/oracle_raster.c:cov3d_from_scale_rot)
__device__ __forceinline__ void cov3d_from_scale_rot(const float* __restrict__ s3, float mod,
                                                     const float4 q, float* c6) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    const float sx = mul_(s3[0], mod), sy = mul_(s3[1], mod), sz = mul_(s3[2], mod);
    const float yy = mul_(y, y), zz = mul_(z, z), xz = mul_(x, z), rx = mul_(r, x), rz = mul_(r, z);
    float t;
    t = add_(yy, zz);            const float R00 = sub_(1.0f, add_(t, t));
    t = fma_(x, y, -rz);         const float R01 = add_(t, t);
    t = fma_(r, y, xz);          const float R02 = add_(t, t);
    t = fma_(x, y, rz);          const float R10 = add_(t, t);
    t = fma_(x, x, zz);          const float R11 = sub_(1.0f, add_(t, t));
    t = fma_(y, z, -rx);         const float R12 = add_(t, t);
    t = fma_(-r, y, xz);         const float R20 = add_(t, t);
    t = fma_(y, z, rx);          const float R21 = add_(t, t);
    t = fma_(x, x, yy);          const float R22 = sub_(1.0f, add_(t, t));
    const float z00 = mul_(0.0f, R00), z11 = mul_(0.0f, R11), z21 = mul_(0.0f, R21);
    const float m00 = fma_(0.0f, R02, fma_(0.0f, R01, mul_(sx, R00)));
    const float m01 = fma_(0.0f, R02, fma_(sy, R01, z00));
    const float m02 = fma_(sz, R02, fma_(0.0f, R01, z00));
    const float m10 = fma_(0.0f, R12, fma_(sx, R10, z11));
    const float m11 = fma_(0.0f, R12, fma_(0.0f, R10, mul_(sy, R11)));
    const float m12 = fma_(sz, R12, fma_(0.0f, R10, z11));
    const float m20 = fma_(0.0f, R22, fma_(sx, R20, z21));
    const float m21 = fma_(0.0f, R22, fma_(0.0f, R20, mul_(sy, R21)));
    const float m22 = fma_(sz, R22, fma_(0.0f, R20, z21));
    c6[0] = dot3_(m00, m00, m01, m01, m02, m02);
    c6[1] = dot3_(m00, m10, m01, m11, m02, m12);
    c6[2] = dot3_(m00, m20, m01, m21, m02, m22);
    c6[3] = dot3_(m10, m10, m11, m11, m12, m12);
    c6[4] = dot3_(m10, m20, m11, m21, m12, m22);
    c6[5] = dot3_(m20, m20, m21, m21, m22, m22);
}

struct ProjParams {
    int P, S, D, M, W, H, gx, gy, recf, ng;
    const float *means3D, *shs, *colors_precomp, *features, *opacities, *scales, *rotations,
        *cov3D_precomp, *viewmatrix, *projmatrix, *campos;
    float scale_modifier, tan_fovx, tan_fovy, focal_x, focal_y;
    int prefiltered, antialiasing;
    float* rec;
    uint32_t* tiles_touched;
    uint8_t* clamped;
    int* radii;
    float* out_weights;
    GeomHeader* header;
    uint32_t *sort_keys, *sort_vals;      // depth-sort input (radix_sort.cu)
    uint2* rects;                         // packed tile rectangles (binning.cu)
    uint2* brects;                        // packed block rectangles (compositor pre-filter, common.cuh block_rect)
    const float* filter_3d;               // F3D: [P] Mip-Splatting 3D filter sizes (last: the other fields keep their offsets)
};

#define PROJ_THREADS 128
// Cooperative, coalesced load of the block's [nvalid][rowf] float slab into a transposed shared
// slab s[k * (PROJ_THREADS + 1) + t] (conflict-free column access by thread t).
__device__ __forceinline__ void load_rows_transposed(float* s, const float* __restrict__ src, int nvalid, int rowf) {
    const int total = nvalid * rowf;
    if ((rowf & 3) == 0) {
        const float4* src4 = reinterpret_cast<const float4*>(src);
        for (int i4 = threadIdx.x; i4 < total / 4; i4 += PROJ_THREADS) {
            const float4 v = src4[i4];
            const int i = 4 * i4, t = i / rowf, k = i - t * rowf;
            s[(k + 0) * (PROJ_THREADS + 1) + t] = v.x; s[(k + 1) * (PROJ_THREADS + 1) + t] = v.y;
            s[(k + 2) * (PROJ_THREADS + 1) + t] = v.z; s[(k + 3) * (PROJ_THREADS + 1) + t] = v.w;
        }
    } else {
        for (int i = threadIdx.x; i < total; i += PROJ_THREADS) {
            const int t = i / rowf, k = i - t * rowf;
            s[k * (PROJ_THREADS + 1) + t] = src[i];
        }
    }
}

// F3D: Mip-Splatting's 3D filter (common.cuh filter3d_fold) — the Gaussian is projected with the dilated scales s' and
// its opacity is o coef; cov3D_precomp is refused by the caller.
// RD (ray-depth mode): the record's appended group holds the depth plane p = conic (T0 Sigma w_z, T1 Sigma w_z), the
// gradient of camera z's conditional mean given the screen position (w_z: the view matrix's camera-z column).
template <bool F3D = false, bool RD = false>
__global__ void __launch_bounds__(PROJ_THREADS) project_kernel(const ProjParams p) {
    extern __shared__ __align__(16) float sSH[];   // SH slab ([3M][PROJ_THREADS + 1] transposed, or row-major), later the record slab
    __shared__ float sV[16], sPr[16], sCam[3];
    if (threadIdx.x < 16) { sV[threadIdx.x] = p.viewmatrix[threadIdx.x]; sPr[threadIdx.x] = p.projmatrix[threadIdx.x]; }
    if (threadIdx.x < 3) sCam[threadIdx.x] = p.campos[threadIdx.x];
    __syncthreads();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    bool alive = idx < p.P;
    float px = 0.f, py = 0.f, pz = 0.f, tz = 1.f;
    if (alive) {
        p.radii[idx] = 0;
        p.tiles_touched[idx] = 0;
        p.out_weights[idx] = 0.0f;
        p.sort_vals[idx] = (uint32_t)idx;
        px = p.means3D[3 * (size_t)idx]; py = p.means3D[3 * (size_t)idx + 1]; pz = p.means3D[3 * (size_t)idx + 2];
        tz = xform_row_(sV, 2, px, py, pz);
        if (tz <= 0.2f) {                              // auxiliary.h:154 (x/y frustum test is disabled there)
            if (p.prefiltered) { printf("Point is filtered although prefiltered is set. This shouldn't happen!"); __trap(); }
            alive = false;
        }
    }
    // SH rows ([M][3] floats, 192 B at M=16 = 3/4 of the kernel's input bytes) are staged in shared memory.  The
    // CTA's rows are ONE contiguous 24 KB slab, so a single TMA-unit bulk copy (cp.async.bulk -> UBLKCP) moves it
    // with no per-thread instructions and signals an mbarrier; it is issued as soon as the depth cull is known and
    // overlaps the covariance / projection math below.  Blocks whose Gaussians are all behind the camera skip it.
    // (Rows that are not a multiple of 16 B — SH degree 0 / 2 — or a ragged, unaligned tail fall back to 4-byte
    // LDGSTS copies into a transposed slab.)
    __shared__ __align__(8) uint64_t sBar;
    bool slab_loaded = false, slab_bulk = false;
    const int rowf = 3 * p.M;
    if (p.colors_precomp == nullptr) {
        const int block_base = blockIdx.x * PROJ_THREADS;
        const int nvalid = min(PROJ_THREADS, p.P - block_base);
        const float* src = p.shs + (size_t)block_base * rowf;
        const unsigned bytes = (unsigned)nvalid * (unsigned)rowf * 4u;
        slab_bulk = (rowf & 3) == 0 && (bytes & 15u) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
        if (threadIdx.x == 0 && slab_bulk) { mbar_init(&sBar, 1); fence_proxy_async_smem(); }
        slab_loaded = __syncthreads_or(alive) != 0;
        if (slab_loaded) {
            if (slab_bulk) {
                if (threadIdx.x == 0) { mbar_arrive_expect_tx(&sBar, bytes); bulk_copy_g2s(sSH, src, bytes, &sBar); }
            } else {
                load_rows_transposed_async(sSH, PROJ_THREADS + 1, src, nvalid, rowf, PROJ_THREADS);
                cp_async_commit();
            }
        }
    }
    float pix_x = 0.f, pix_y = 0.f, con_a = 0.f, con_b = 0.f, con_c = 0.f, aa_rho = 1.f, f3d_coef = 1.f;
    float pl_x = 0.f, pl_y = 0.f;                      // RD: the depth plane
    int my_radius = 0, x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    if (alive) {
        const float hx = xform_row_(sPr, 0, px, py, pz);
        const float hy = xform_row_(sPr, 1, px, py, pz);
        const float hw = xform_row_(sPr, 3, px, py, pz);
        const float p_w = rcp_(add_(hw, 0.0000001f));
        const float projx = mul_(hx, p_w), projy = mul_(hy, p_w);
        float c6[6];
        if (p.cov3D_precomp) {
#pragma unroll
            for (int i = 0; i < 6; ++i) c6[i] = p.cov3D_precomp[6 * (size_t)idx + i];
        } else {
            const float4 q = *reinterpret_cast<const float4*>(p.rotations + 4 * (size_t)idx);
            if constexpr (F3D) {
                float s3[3] = {p.scales[3 * (size_t)idx], p.scales[3 * (size_t)idx + 1], p.scales[3 * (size_t)idx + 2]};
                f3d_coef = filter3d_fold(s3, p.filter_3d[idx]);
                cov3d_from_scale_rot(s3, p.scale_modifier, q, c6);
            } else {
                const float s3[3] = {p.scales[3 * (size_t)idx], p.scales[3 * (size_t)idx + 1], p.scales[3 * (size_t)idx + 2]};
                cov3d_from_scale_rot(s3, p.scale_modifier, q, c6);
            }
        }
        // computeCov2D (forward.cu:74-113), association as compiled
        const float tx = xform_row_(sV, 0, px, py, pz), ty = xform_row_(sV, 1, px, py, pz);
        const float limx = mul_(p.tan_fovx, 1.3f), limy = mul_(p.tan_fovy, 1.3f);
        const float cxz = fminf(fmaxf(div_(tx, tz), -limx), limx);
        const float cyz = fminf(fmaxf(div_(ty, tz), -limy), limy);
        const float tz2 = mul_(tz, tz);
        const float j00 = div_(p.focal_x, tz), j11 = div_(p.focal_y, tz);
        const float j02 = div_(mul_(mul_(tz, -cxz), p.focal_x), tz2);
        const float j12 = div_(mul_(mul_(tz, -cyz), p.focal_y), tz2);
        float T0[3], T1[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float w0 = sV[4 * k + 0], w1 = sV[4 * k + 1], w2 = sV[4 * k + 2];
            T0[k] = fma_(w2, j02, fma_(w0, j00, mul_(0.0f, w1)));
            T1[k] = fma_(w2, j12, fma_(0.0f, w0, mul_(w1, j11)));
        }
        const float a0 = dot3_(T0[0], c6[0], T0[1], c6[1], T0[2], c6[2]);
        const float a1 = dot3_(T0[0], c6[1], T0[1], c6[3], T0[2], c6[4]);
        const float a2 = dot3_(T0[0], c6[2], T0[1], c6[4], T0[2], c6[5]);
        const float b0 = dot3_(T1[0], c6[0], T1[1], c6[1], T1[2], c6[2]);
        const float b1 = dot3_(T1[0], c6[1], T1[1], c6[3], T1[2], c6[4]);
        const float b2 = dot3_(T1[0], c6[2], T1[1], c6[4], T1[2], c6[5]);
        const float cov_a0 = dot3_(T0[0], a0, T0[1], a1, T0[2], a2);
        const float cov_c0 = dot3_(T1[0], b0, T1[1], b1, T1[2], b2);
        const float cov_a = add_(cov_a0, 0.3f);
        const float cov_c = add_(cov_c0, 0.3f);
        const float cov_b = dot3_(T0[0], b0, T0[1], b1, T0[2], b2);
        const float det = fma_(cov_a, cov_c, -mul_(cov_b, cov_b));
        if (det == 0.0f) {
            alive = false;
        } else {
            if (p.antialiasing) {                      // (uniform) rho = sqrt(max(det0 / det, 2.5e-5)), r = 0 for det0 <= 0
                const float det0 = fma_(cov_a0, cov_c0, -mul_(cov_b, cov_b));
                aa_rho = sqrt_(fmaxf(det0 > 0.0f ? div_(det0, det) : 0.0f, 2.5e-5f));
            }
            const float det_inv = rcp_(det);
            con_a = mul_(cov_c, det_inv); con_b = mul_(cov_b, -det_inv); con_c = mul_(cov_a, det_inv);
            if constexpr (RD) {                        // c = (T0 Sigma w_z, T1 Sigma w_z) from the a, b products, p = conic c
                const float cu = fmaf(a2, sV[10], fmaf(a1, sV[6], a0 * sV[2]));
                const float cv = fmaf(b2, sV[10], fmaf(b1, sV[6], b0 * sV[2]));
                pl_x = fmaf(con_b, cv, con_a * cu);
                pl_y = fmaf(con_c, cv, con_b * cu);
            }
            const float mid = mul_(add_(cov_a, cov_c), 0.5f);
            const float disc = sqrt_(fmaxf(fma_(mid, mid, -det), 0.1f));
            const float lam = fmaxf(add_(mid, disc), sub_(mid, disc));
            my_radius = (int)ceilf(mul_(sqrt_(lam), 3.0f));
            pix_x = (float)(fma((double)projx + 1.0, (double)p.W, -1.0) * 0.5);   // ndc2Pix, auxiliary.h:41-44
            pix_y = (float)(fma((double)projy + 1.0, (double)p.H, -1.0) * 0.5);
            get_rect(pix_x, pix_y, my_radius, p.gx, p.gy, x0, y0, x1, y1);
            if ((x1 - x0) * (y1 - y0) == 0) alive = false;
        }
    }
    float rgb[3] = {0.f, 0.f, 0.f};
    unsigned cl = 0;                                   // clamped channels; kComposited is set by the forward compositor
    if (p.colors_precomp == nullptr) {
        if (slab_loaded) {
            if (slab_bulk) {
                mbar_wait(&sBar, 0);                       // all transaction bytes of the slab have landed
                // row-major slab: this thread's row as 16-byte vectors (LDS.128: 4 consecutive rows span all banks)
                if (alive) sh_to_rgb(p.D, px, py, pz, sCam, sSH + (size_t)threadIdx.x * rowf, 0, rgb, cl);
            } else {
                cp_async_wait_all();
                __syncthreads();
                if (alive) sh_to_rgb(p.D, px, py, pz, sCam, sSH + threadIdx.x, PROJ_THREADS + 1, rgb, cl);
            }
        }
    } else if (alive) {
        rgb[0] = p.colors_precomp[3 * (size_t)idx]; rgb[1] = p.colors_precomp[3 * (size_t)idx + 1]; rgb[2] = p.colors_precomp[3 * (size_t)idx + 2];
    }
    {   // which depth-key bits vary across the visible Gaussians (drives radix pass skipping)
        const uint32_t bits = __float_as_uint(tz);
        const uint32_t o = __reduce_or_sync(0xffffffffu, alive ? bits : 0u);
        const uint32_t no = __reduce_or_sync(0xffffffffu, alive ? ~bits : 0u);
        if ((threadIdx.x & 31) == 0 && (o | no)) { atomicOr(&p.header->depth_or, o); atomicOr(&p.header->depth_nor, no); }
    }
    if (idx < p.P) {   // depth-sort key + packed tile rectangle {x0 | y0 << 16, w | h << 16}; culled: empty rectangle
        p.sort_keys[idx] = alive ? __float_as_uint(tz) : 0u;
        p.rects[idx] = alive ? make_uint2((uint32_t)x0 | ((uint32_t)y0 << 16), (uint32_t)(x1 - x0) | ((uint32_t)(y1 - y0) << 16))
                             : make_uint2(0u, 0u);
    }
    // ---- packed record row: staged in shared memory (the SH slab is dead by now), written back by ONE TMA bulk store ---
    // A thread writing its own 64-112 B row straight to global memory issues 4-7 STG.128 whose 32 lanes are 64-112 B
    // apart: every instruction touches 32 half-used sectors and the kernel was bound by the L1/TEX pipeline, not by
    // HBM.  The CTA's rows are one contiguous slab; rows of
    // culled Gaussians are written as zeros (nothing ever reads them: they are in no tile list).
    const int rec4n = p.recf >> 2;
    float4* srow = reinterpret_cast<float4*>(sSH) + (size_t)threadIdx.x * rec4n;
    __syncthreads();                                   // every thread is done with the SH slab
    if (alive) {
        // antialiased mode: the compensated opacity o * rho is the opacity of everything downstream (3D filter: o coef rho)
        const float o = F3D ? mul_(p.opacities[idx], f3d_coef) : p.opacities[idx];
        const float op = p.antialiasing ? mul_(o, aa_rho) : o;
        p.brects[idx] = block_rect(pix_x, pix_y, con_a, con_b, con_c, op);
        srow[0] = make_float4(pix_x, pix_y, con_a, con_b);
        srow[1] = make_float4(con_c, op, tz, __int_as_float(my_radius));
        // channels {r,g,b,f0..}, zero padded
        const float* f = p.features + (size_t)idx * p.S;
        for (int g = 0; g < p.ng; ++g) {
            float v[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int c = 4 * g + k;
                v[k] = c < 3 ? rgb[c] : (c - 3 < p.S ? f[c - 3] : 0.0f);
            }
            srow[2 + g] = make_float4(v[0], v[1], v[2], v[3]);
        }
        if constexpr (RD) srow[2 + p.ng] = make_float4(pl_x, pl_y, 0.f, 0.f);
        p.radii[idx] = my_radius;
        p.tiles_touched[idx] = (uint32_t)((y1 - y0) * (x1 - x0));
        p.clamped[idx] = (uint8_t)cl;
    } else if (idx < p.P) {
        for (int g = 0; g < rec4n; ++g) srow[g] = make_float4(0.f, 0.f, 0.f, 0.f);
        p.clamped[idx] = 0;                            // culled: never composited
    }
    fence_proxy_async_smem();                          // this thread's shared-memory stores -> visible to the bulk-copy engine
    __syncthreads();
    if (threadIdx.x == 0) {
        const int block_base = blockIdx.x * PROJ_THREADS;
        const int nvalid = min(PROJ_THREADS, p.P - block_base);
        bulk_copy_s2g(p.rec + (size_t)block_base * p.recf, sSH, (unsigned)nvalid * (unsigned)p.recf * 4u);
        bulk_wait_read_all();                          // the slab must stay alive until the engine has read it
    }
}

// ---- chained (decoupled look-back) inclusive scan of tiles_touched -> point_offsets ----------
// One pass over the data, block order fixed by an atomic ticket.  state[b]: bits 31..30 flag
// (1 = aggregate, 2 = inclusive prefix), bits 29..0 value.
#define SCAN_THREADS 256
#define SCAN_PER_THREAD (R3DG_SCAN_ITEMS / SCAN_THREADS)
__global__ void __launch_bounds__(SCAN_THREADS) scan_kernel(int P, const uint32_t* __restrict__ in,
                                                            uint32_t* __restrict__ out,
                                                            volatile uint32_t* state, GeomHeader* header) {
    __shared__ uint32_t s_block, s_warp[SCAN_THREADS / 32], s_prefix;
    if (threadIdx.x == 0) s_block = atomicAdd(&header->scan_ticket, 1u);
    __syncthreads();
    const uint32_t b = s_block;
    const int base = b * R3DG_SCAN_ITEMS + threadIdx.x * SCAN_PER_THREAD;
    uint32_t v[SCAN_PER_THREAD], sum = 0;
    if (base + SCAN_PER_THREAD <= P) {           // 2 x 16 B vector loads (base is a multiple of 8 elements)
        const uint4* in4 = reinterpret_cast<const uint4*>(in + base);
#pragma unroll
        for (int q = 0; q < SCAN_PER_THREAD / 4; ++q) { const uint4 t = in4[q]; v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w; }
    } else {
#pragma unroll
        for (int i = 0; i < SCAN_PER_THREAD; ++i) v[i] = base + i < P ? in[base + i] : 0u;
    }
#pragma unroll
    for (int i = 0; i < SCAN_PER_THREAD; ++i) sum += v[i];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += t; }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < SCAN_THREADS / 32 ? s_warp[lane] : 0u, wi = w;
#pragma unroll
        for (int d = 1; d < 8; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= d) wi += t; }
        if (lane < SCAN_THREADS / 32) s_warp[lane] = wi - w;            // exclusive warp offsets
        const uint32_t total = __shfl_sync(0xffffffffu, wi, SCAN_THREADS / 32 - 1);
        // warp-parallel decoupled look-back: lane i inspects block b-1-i, 32 predecessors per round
        uint32_t prefix = 0;
        if (b == 0) {
            if (lane == 0) st_relaxed_gpu(const_cast<uint32_t*>(state), total | 0x80000000u);
        } else {
            if (lane == 0) st_relaxed_gpu(const_cast<uint32_t*>(state) + b, total | 0x40000000u);
            int t = (int)b - 1;
            while (true) {
                const uint32_t sv = (t - lane >= 0) ? ld_relaxed_gpu(const_cast<const uint32_t*>(state) + (t - lane)) : 0x80000000u;
                const unsigned ready = __ballot_sync(0xffffffffu, (sv >> 30) != 0u);
                const unsigned incl = __ballot_sync(0xffffffffu, (sv >> 30) == 2u);
                // usable run: consecutive ready lanes from lane 0, cut at the first inclusive one
                const int n_ready = __ffs(~ready) - 1 < 0 ? 32 : __ffs(~ready) - 1;
                const int first_inc = incl ? __ffs(incl) - 1 : 32;
                const int take = first_inc < n_ready ? first_inc + 1 : n_ready;
                uint32_t v = lane < take ? (sv & 0x3fffffffu) : 0u;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                prefix += v;
                if (first_inc < n_ready) break;
                t -= take;
            }
            if (lane == 0) st_relaxed_gpu(const_cast<uint32_t*>(state) + b, (prefix + total) | 0x80000000u);
        }
        if (lane == 0) {
            s_prefix = prefix;
            if ((int)b == (P + R3DG_SCAN_ITEMS - 1) / R3DG_SCAN_ITEMS - 1) header->num_rendered = prefix + total;
        }
    }
    __syncthreads();
    uint32_t run = s_prefix + s_warp[warp] + (inc - sum);
#pragma unroll
    for (int i = 0; i < SCAN_PER_THREAD; ++i) { run += v[i]; v[i] = run; }
    if (base + SCAN_PER_THREAD <= P) {
        uint4* out4 = reinterpret_cast<uint4*>(out + base);
#pragma unroll
        for (int q = 0; q < SCAN_PER_THREAD / 4; ++q) out4[q] = make_uint4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    } else {
#pragma unroll
        for (int i = 0; i < SCAN_PER_THREAD; ++i) if (base + i < P) out[base + i] = v[i];
    }
}

// The same coarse LPT order as the tile order (binning.cu, bin_starts) for the backward compositor's CTAs, by what the forward pass measured: keys[c] = entries the
// busiest warp of half-tile CTA c composited = exactly the iterations its backward twin will run.  List length is a poor
// predictor there (a dense tile saturates after a fraction of its list): ordered by it, heavy backward CTAs started
// late and finished last (the per-warp timing study of commit 072299e, DESIGN.md §4.2).
__global__ void __launch_bounds__(1024) cta_order_kernel(int n, const uint32_t* __restrict__ keys, uint32_t* __restrict__ order) {
    __shared__ uint32_t s_max, s_cnt[64], s_cur[64];
    const int tid = threadIdx.x;
    if (tid == 0) s_max = 0;
    if (tid < 64) s_cnt[tid] = 0;
    __syncthreads();
    uint32_t m = 0;
    for (int t = tid; t < n; t += 1024) m = max(m, keys[t]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) atomicMax(&s_max, m);
    __syncthreads();
    const uint32_t mx = s_max;
    const int shift = mx < 64 ? 0 : (32 - __clz(mx)) - 6;            // bucket = key >> shift in [0, 63]
    for (int t = tid; t < n; t += 1024) atomicAdd(&s_cnt[min(63u, keys[t] >> shift)], 1u);
    __syncthreads();
    if (tid == 0) { uint32_t acc = 0; for (int b = 63; b >= 0; --b) { s_cur[b] = acc; acc += s_cnt[b]; } }   // descending
    __syncthreads();
    for (int t = tid; t < n; t += 1024) order[atomicAdd(&s_cur[min(63u, keys[t] >> shift)], 1u)] = (uint32_t)t;
}

__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D,
                                    const float* __restrict__ viewmatrix, uint8_t* __restrict__ present) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float tz = xform_row_(viewmatrix, 2, means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]);
    present[idx] = tz > 0.2f ? 1 : 0;
}

// ---- host launchers -----------------------------------------------------------------------
int launch_projection(const r3dg_raster_fwd_args& a, const RasterBuffers& b, int v, cudaStream_t stream) {
    ProjParams p;
    float tan_fovx = a.tan_fovx, tan_fovy = a.tan_fovy, cx = a.cx, cy = a.cy;
    view_cam(b.V, a.view_cams, v, tan_fovx, tan_fovy, cx, cy);
    const size_t r = (size_t)v * a.P;                 // view v's rows of the per-view inputs and outputs
    p.P = a.P; p.S = a.S; p.D = a.D; p.M = a.M; p.W = a.W; p.H = a.H;
    p.gx = b.gx; p.gy = b.gy;
    p.recf = b.recf; p.ng = num_groups(a.S);
    p.means3D = a.means3D; p.shs = a.shs; p.opacities = a.opacities; p.scales = a.scales; p.rotations = a.rotations;
    p.cov3D_precomp = a.cov3D_precomp;
    p.colors_precomp = a.colors_precomp && a.colors_per_view ? a.colors_precomp + 3 * r : a.colors_precomp;
    p.features = a.features && a.features_per_view ? a.features + (size_t)a.S * r : a.features;
    p.viewmatrix = a.viewmatrix + 16 * v; p.projmatrix = a.projmatrix + 16 * v; p.campos = a.campos + 3 * v;
    p.scale_modifier = a.scale_modifier; p.tan_fovx = tan_fovx; p.tan_fovy = tan_fovy;
    p.focal_y = a.H / (2.0f * tan_fovy);              // rasterizer_impl.cu:232-233
    p.focal_x = a.W / (2.0f * tan_fovx);
    p.prefiltered = a.prefiltered; p.antialiasing = a.antialiasing;
    p.rec = b.rec; p.tiles_touched = b.tiles_touched;
    p.clamped = b.clamped; p.radii = a.radii + r; p.out_weights = a.out_weights + r;
    p.header = b.header;
    p.sort_keys = (uint32_t*)(b.sort + b.sort_layout.keys_a);
    p.sort_vals = (uint32_t*)(b.sort + b.sort_layout.vals_a);
    p.rects = b.rects; p.brects = b.brects;
    p.filter_3d = a.filter_3d;
    // dynamic shared memory: the SH slab (transposed fallback layout is the larger one), reused for the record slab
    size_t sh_smem = a.shs ? (size_t)3 * a.M * (PROJ_THREADS + 1) * sizeof(float) : 0;
    const size_t rec_smem = (size_t)PROJ_THREADS * b.recf * sizeof(float);
    if (rec_smem > sh_smem) sh_smem = rec_smem;
    const int blocks = (a.P + PROJ_THREADS - 1) / PROJ_THREADS;
    if (a.ray_depth) {
        if (a.filter_3d) project_kernel<true, true><<<blocks, PROJ_THREADS, sh_smem, stream>>>(p);
        else project_kernel<false, true><<<blocks, PROJ_THREADS, sh_smem, stream>>>(p);
    } else if (a.filter_3d) {
        project_kernel<true><<<blocks, PROJ_THREADS, sh_smem, stream>>>(p);
    } else {
        project_kernel<<<blocks, PROJ_THREADS, sh_smem, stream>>>(p);
    }
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

// Debug only (r3dg_raster_debug_copy id 8): the reference's geomState.point_offsets, the inclusive
// scan of tiles_touched in Gaussian-index order (rasterizer_impl.cu:288).  The hot path no longer
// needs it.  `state` holds P / R3DG_SCAN_ITEMS + 2 words, `ticket_header` a zeroed GeomHeader.
int launch_point_offsets(int P, const uint32_t* tiles_touched, uint32_t* out, uint32_t* state,
                         GeomHeader* ticket_header, cudaStream_t stream) {
    const int nscan = (P + R3DG_SCAN_ITEMS - 1) / R3DG_SCAN_ITEMS;
    R3DG_CUDA_TRY(cudaMemsetAsync(state, 0, (size_t)(nscan + 1) * 4, stream));
    R3DG_CUDA_TRY(cudaMemsetAsync(ticket_header, 0, sizeof(GeomHeader), stream));
    scan_kernel<<<nscan, SCAN_THREADS, 0, stream>>>(P, tiles_touched, out, (volatile uint32_t*)state, ticket_header);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_cta_order(const uint32_t* work, uint32_t* order, int n, cudaStream_t stream) {
    cta_order_kernel<<<1, 1024, 0, stream>>>(n, work, order);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                        cudaStream_t stream) {
    if (P <= 0) return 0;
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, viewmatrix, present);
    R3DG_CUDA_TRY(cudaGetLastError());
    return 0;
}

}  // namespace r3dg
