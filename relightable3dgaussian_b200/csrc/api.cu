// C ABI of libr3dg_b200.so (declared in include/r3dg_b200.h).  Orchestration only: all device
// work is enqueued on the caller's stream; there is no host synchronisation, no allocation and
// no global state besides the per-device SM-count cache.
#include <cstdio>
#include <cstring>
#include <vector>
#include "common.cuh"
#include "detacc.cuh"
#include "kernels.h"

using namespace r3dg;

int r3dg::num_sms() {
    static int per_device[kMaxDevices] = {0};      // the caller may drive several GPUs from one process
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 132;   // H100 SXM
    if (per_device[dev] == 0) {
        int n = 0;
        per_device[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
    }
    return per_device[dev];
}

namespace {
// ---- optional stage profiler: CUDA events recorded on the launching stream between stages ----
enum { ST_PROJECT = 0, ST_DEPTH_SORT, ST_BIN_COUNT, ST_BIN_OFFSETS, ST_BIN_SCATTER, ST_COMPOSITE, ST_NORMAL, ST_COMPOSITE_BWD,
       ST_PROJECT_BWD, ST_COUNT };
struct Prof {
    bool on = false;
    int max_calls = 0, fwd_calls = 0, bwd_calls = 0;
    std::vector<cudaEvent_t> ev;      // [max_calls][ST_COUNT + 2]  (fwd: 0..7 boundaries, bwd: 8..10)
    cudaEvent_t& at(int call, int i) { return ev[(size_t)call * (ST_COUNT + 2) + i]; }
} g_prof;
unsigned long long g_launches = 0;
inline void prof_mark(bool fwd, int i, cudaStream_t s) {
    if (!g_prof.on) return;
    const int call = fwd ? g_prof.fwd_calls : g_prof.bwd_calls;
    if (call >= g_prof.max_calls) return;
    cudaEventRecord(g_prof.at(call, i), s);
}
// The kernels read each quaternion (rotations) and write each dL_drotations row as one float4: a [P,4] array whose
// base is not 16-byte aligned (a contiguous view at an odd storage offset) is refused before anything is launched.
inline bool misaligned16(const void* p) { return p && (reinterpret_cast<uintptr_t>(p) & 15u) != 0; }

// ---- the rasterizer's work buffers: regions in this order, each 256-byte aligned ---------------------------------
// V views: V rows per Gaussian (row v * P + g), one header and one depth-sort region per view.  V = 1 is the one-view
// layout.  Ray-depth mode: records and gradient rows one float4 wider (common.cuh rec_floats).
struct GeomLayout {
    size_t header, rec, tiles_touched, rects, brects, clamped, scan_state, sort, sort_stride, grad, total;
    int recf;
    SortLayout sl;
    GeomLayout(int P, int S, int V = 1, bool ray_depth = false) : recf(rec_floats(S, ray_depth)), sl(P) {
        const size_t R = (size_t)V * P;
        sort_stride = align_up(sl.total, 256);
        size_t off = 0;
        header = off;        off = align_up(off + V * sizeof(GeomHeader), 256);
        rec = off;           off = align_up(off + R * recf * 4, 256);
        tiles_touched = off; off = align_up(off + R * 4, 256);
        rects = off;         off = align_up(off + R * 8, 256);                 // packed tile rectangles
        brects = off;        off = align_up(off + R * 8, 256);                 // packed block rectangles (block_rect())
        clamped = off;       off = align_up(off + R, 256);
        scan_state = off;    off = align_up(off + ((size_t)P / R3DG_SCAN_ITEMS + 2) * 4, 256);
        sort = off;          off = align_up(off + V * sort_stride, 256);        // depth sort of the Gaussians, per view
        grad = off;          off = align_up(off + R * recf * 4, 256);           // backward scratch
        // ray-depth mode: one more 256-byte block, so that a ray-depth buffer is always larger than a default one of
        // the same shape and a host layer can tell the mode of a geometry buffer from its size (_C_raster.py)
        if (ray_depth) off += 256;
        total = off;
    }
};

// V views: V images stacked as one tall tile grid (view v owns tile rows [v * gy, (v + 1) * gy)); the binning scratch
// (slab sums, count matrix) is per view and reused by the views one after the other.
// Depth statistics: two more regions behind the default layout (whose offsets they leave as they are), so that such a
// buffer is always larger than a default one of the same shape: the median entry's list position per pixel, and per
// view the largest |d| of an accepted entry (the deterministic backward's scale).
struct ImgLayout {
    size_t final_T, n_contrib, ranges, tile_order, bwd_work, bwd_order, slab_sum, bin_matrix, median_pos, depth_bound, total;
    int gx, gy, max_chunks;
    ImgLayout(int W, int H, int V = 1, bool depth_stats = false)
        : gx((W + R3DG_TILE - 1) / R3DG_TILE), gy((H + R3DG_TILE - 1) / R3DG_TILE) {
        const size_t HW = (size_t)W * H * V, T = (size_t)gx * gy, VT = T * V;
        max_chunks = bin_max_chunks(T);
        size_t off = 0;
        final_T = off;   off = align_up(off + HW * 4, 256);
        n_contrib = off; off = align_up(off + HW * 4, 256);
        ranges = off;    off = align_up(off + VT * 8, 256);
        tile_order = off; off = align_up(off + VT * 4, 256);      // tiles by descending list length
        bwd_work = off;  off = align_up(off + 2 * VT * 4, 256);   // per half-tile CTA: entries its busiest warp composited (forward)
        bwd_order = off; off = align_up(off + 2 * VT * 4, 256);  // half-tile CTAs by descending bwd_work (backward launch order)
        slab_sum = off;  off = align_up(off + T * 4 * ((R3DG_BIN_MAX_CHUNKS + 511) / 512), 256);   // per 512-chunk slab
        bin_matrix = off; off = align_up(off + ((size_t)max_chunks + 1) * T * 4, 256);   // + the row of list ends
        median_pos = off; depth_bound = align_up(off + HW * 4, 256);
        if (depth_stats) off = align_up(depth_bound + (size_t)V * 4, 256);
        total = off;
    }
};

// Binning buffer (capacity-sized, speculative): the per-tile depth-sorted Gaussian lists (reference
// binningState.point_list) plus one byte per instance for each of
//   bmask: bit b = 8x4 pixel block b of the instance's tile may be touched by the Gaussian (written by bin_scatter
//          with block_mask_of_rect: the conservative block-rectangle test evaluated ONCE per instance instead of by 8 warps);
//   cmask: bit b = block b actually composited the instance in the forward pass (some pixel accepted it).  The
//          backward compositor visits exactly the cmask entries of its block, nothing else.
// 6 B per instance instead of the reference's 24 B + sort temp.
struct BinLayout {
    size_t point_list, bmask, cmask, total;
    long long capacity;
    BinLayout(long long cap) : capacity(cap) {
        size_t off = 0;
        point_list = off; off = align_up(off + (size_t)cap * 4, 256);
        bmask = off;      off = align_up(off + (size_t)cap, 256);
        cmask = off;      off = align_up(off + (size_t)cap, 256);
        total = off;
    }
};
// largest capacity (a multiple of 64 instances) whose layout fits in `bytes`; r3dg_raster_binning_bytes is its inverse
long long bin_capacity_for_bytes(size_t bytes) { return bytes < 768 + 384 ? 0 : (long long)((bytes - 768) / 6 / 64 * 64); }
size_t bin_bytes_for_capacity(long long cap) { return (size_t)((cap + 63) / 64 * 64) * 6 + 768; }

// Fills `b` for one call; P = 0 is laid out as P = 1, as r3dg_raster_geom_bytes sizes it.  Returns R3DG_ERR_BAD_ARG
// when a buffer is smaller than its layout or the binning buffer holds no instance, and fills `b` either way
// (r3dg_raster_debug_copy passes SIZE_MAX for the sizes it is not given, and needs the binning only for some ids).
int raster_buffers(int P, int S, int W, int H, void* geom_, size_t geom_bytes, void* img_, size_t img_bytes,
                   void* bin_, size_t bin_bytes, RasterBuffers& b, int V = 1, bool ray_depth = false,
                   bool depth_stats = false) {
    const GeomLayout gl(P < 1 ? 1 : P, S, V, ray_depth);
    const ImgLayout il(W, H, V, depth_stats);
    const BinLayout bl(bin_capacity_for_bytes(bin_bytes));
    char *geom = (char*)geom_, *img = (char*)img_, *bin = (char*)bin_;
    b.header = (GeomHeader*)(geom + gl.header);
    b.rec = (float*)(geom + gl.rec); b.grad = (float*)(geom + gl.grad);
    b.tiles_touched = (uint32_t*)(geom + gl.tiles_touched);
    b.rects = (uint2*)(geom + gl.rects); b.brects = (uint2*)(geom + gl.brects);
    b.clamped = (uint8_t*)(geom + gl.clamped);
    b.sort = geom + gl.sort; b.sort_layout = gl.sl;
    b.final_T = (float*)(img + il.final_T); b.n_contrib = (int*)(img + il.n_contrib);
    b.median_pos = (int*)(img + il.median_pos); b.depth_bound = (uint32_t*)(img + il.depth_bound);   // (depth statistics)
    b.ranges = (uint2*)(img + il.ranges); b.tile_order = (uint32_t*)(img + il.tile_order);
    b.bwd_work = (uint32_t*)(img + il.bwd_work); b.bwd_order = (uint32_t*)(img + il.bwd_order);
    b.slab_sum = (uint32_t*)(img + il.slab_sum); b.bin_matrix = (uint32_t*)(img + il.bin_matrix);
    b.point_list = (uint32_t*)(bin + bl.point_list);
    b.bmask = (uint8_t*)(bin + bl.bmask); b.cmask = (uint8_t*)(bin + bl.cmask);
    b.capacity = bl.capacity;
    b.recf = gl.recf; b.gx = il.gx; b.gy = il.gy; b.tiles = il.gx * il.gy;
    b.chunk_len = bin_chunk_len(P, il.max_chunks);          // one read of R3DG_BIN_MAX_CHUNKS sizes M and the chunks
    b.chunks = (P + b.chunk_len - 1) / b.chunk_len;
    b.V = V; b.P = P; b.sort_stride = gl.sort_stride; b.row_base = 0; b.prev_header = nullptr;
    return geom_bytes < gl.total || img_bytes < il.total || bl.capacity < 1 ? R3DG_ERR_BAD_ARG : 0;
}

// views of one call: 1 for V = 0 or 1, V when 1 < V <= R3DG_MAX_VIEWS with the per-view camera table, 0 (refused)
// otherwise; V * P below 2^30 keeps every row id and per-view count inside 32 bits with room to spare
int views_of(int V, const float* view_cams, int P) {
    if (V <= 1) return V < 0 ? 0 : 1;
    if (V > R3DG_MAX_VIEWS || !view_cams || (long long)V * P >= (1LL << 30)) return 0;
    return V;
}
}  // namespace

RasterBuffers r3dg::view_slice(const RasterBuffers& b, int v) {
    RasterBuffers s = b;
    const size_t r = (size_t)v * b.P;
    s.header = b.header + v;
    s.rec = b.rec + r * b.recf; s.grad = b.grad + r * b.recf;
    s.tiles_touched = b.tiles_touched + r;
    s.rects = b.rects + r; s.brects = b.brects + r;
    s.clamped = b.clamped + r;
    s.sort = b.sort + (size_t)v * b.sort_stride;
    s.ranges = b.ranges + (size_t)v * b.tiles;
    s.row_base = (uint32_t)r;
    s.prev_header = v > 0 ? b.header + v - 1 : nullptr;
    if (b.V > 1) s.tile_order = nullptr;            // built once over the whole tall grid (launch_tile_order)
    return s;
}

extern "C" {

const char* r3dg_version(void) { return "r3dg_b200 0.1 sm_90a"; }

size_t r3dg_raster_geom_bytes(int P, int S) { return GeomLayout(P < 1 ? 1 : P, S).total; }
size_t r3dg_raster_img_bytes(int W, int H) { return ImgLayout(W, H).total; }
size_t r3dg_raster_binning_bytes(long long capacity) { return bin_bytes_for_capacity(capacity < 1 ? 1 : capacity); }
size_t r3dg_raster_img_n_contrib_offset(int W, int H) { return ImgLayout(W, H).n_contrib; }
size_t r3dg_raster_views_geom_bytes(int P, int S, int V) { return GeomLayout(P < 1 ? 1 : P, S, V < 1 ? 1 : V).total; }
size_t r3dg_raster_views_img_bytes(int W, int H, int V) { return ImgLayout(W, H, V < 1 ? 1 : V).total; }
size_t r3dg_raster_views_img_n_contrib_offset(int W, int H, int V) { return ImgLayout(W, H, V < 1 ? 1 : V).n_contrib; }
size_t r3dg_raster_ray_depth_geom_bytes(int P, int S, int V) { return GeomLayout(P < 1 ? 1 : P, S, V < 1 ? 1 : V, true).total; }
size_t r3dg_raster_depth_stats_img_bytes(int W, int H, int V) { return ImgLayout(W, H, V < 1 ? 1 : V, true).total; }
size_t r3dg_raster_fwd_det_bytes(int P) { return align_up((size_t)(P < 1 ? 1 : P) * 8, 256); }
size_t r3dg_raster_bwd_det_bytes(int P, int S) { return det_bytes((size_t)(P < 1 ? 1 : P) * rec_floats(S < 0 ? 0 : S)); }
size_t r3dg_raster_ray_depth_bwd_det_bytes(int P, int S) {
    return det_bytes((size_t)(P < 1 ? 1 : P) * rec_floats(S < 0 ? 0 : S, true));
}
size_t r3dg_raster_bwd_det_absgrad_bytes(int P) { return det_bytes(2 * (size_t)(P < 1 ? 1 : P)); }
size_t r3dg_raster_cam_grad_bytes(int P, int V) {
    return align_up((size_t)(V < 1 ? 1 : V) * kCamGradFloats * cam_grad_blocks(P) * sizeof(float), 256);
}
size_t r3dg_raster_surface_grad_bytes(int W, int H, int V) {
    const size_t v = V < 1 ? 1 : V, hw = (size_t)(W < 1 ? 1 : W) * (H < 1 ? 1 : H);
    return align_up(2 * v * hw * sizeof(float), 256) + align_up(v * 9 * surface_grad_blocks(W, H) * sizeof(float), 256);
}

int r3dg_det_sum_scaled_host(long long n, const float* terms, float anchor, float* out) {
    if (n < 0 || (n > 0 && !terms) || !out) return R3DG_ERR_BAD_ARG;
    const int e = det_scale_exp(det_f32_bits(anchor) & 0x7fffffffu);
    uint64_t lo = 0, mid = 0, hi = 0;
    uint32_t flag = 0;
    for (long long i = 0; i < n; ++i) {
        const DetTerm t = det_term(terms[i], e);
        lo += t.lo; mid += t.mid; hi += t.hi; flag |= t.flag;
    }
    *out = det_value(lo, mid, hi, flag, e);
    return 0;
}
int r3dg_det_sum_host(long long n, const float* terms, float* out) { return r3dg_det_sum_scaled_host(n, terms, 0.0f, out); }

int r3dg_raster_forward(const r3dg_raster_fwd_args* a, r3dg_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!a || a->P < 0 || a->W <= 0 || a->H <= 0 || a->S < 0) return R3DG_ERR_BAD_ARG;
    if (a->S > R3DG_MAX_S_FWD) return R3DG_ERR_UNSUPPORTED;
    if (a->P > 0 && ((a->shs == nullptr) == (a->colors_precomp == nullptr))) return R3DG_ERR_BAD_ARG;
    if (a->P > 0 && (a->cov3D_precomp == nullptr) && (a->scales == nullptr || a->rotations == nullptr)) return R3DG_ERR_BAD_ARG;
    if (misaligned16(a->rotations)) return R3DG_ERR_BAD_ARG;
    if (a->shs && a->M > 16) return R3DG_ERR_UNSUPPORTED;
    if (a->filter_3d && a->cov3D_precomp) return R3DG_ERR_BAD_ARG;       // the 3D filter is defined on scales
    if (a->depth_stats && (!a->out_depth2 || !a->out_median_depth)) return R3DG_ERR_BAD_ARG;
    const int V = views_of(a->V, a->view_cams, a->P);
    if (V == 0) return R3DG_ERR_BAD_ARG;
    RasterBuffers b;
    int rc = raster_buffers(a->P, a->S, a->W, a->H, a->geom, a->geom_bytes, a->img, a->img_bytes, a->binning,
                            a->binning_bytes, b, V, a->ray_depth != 0, a->depth_stats != 0);
    if (rc != 0) return rc;
    if (a->deterministic && (!a->det_work || a->det_work_bytes < r3dg_raster_fwd_det_bytes(V * a->P))) return R3DG_ERR_BAD_ARG;
    if (a->P > 0) {                                       // the binning's limits, before any launch
        if ((rc = check_binning_limits(b)) != 0) return rc;
    } else if (V > 1 && (b.gx > 65535 || b.gy > 65535 || b.tiles > 65535)) {
        return R3DG_ERR_UNSUPPORTED;                      // (P == 0: only the tile order of several views runs)
    }
    R3DG_CUDA_TRY(cudaMemsetAsync(b.header, 0, V * sizeof(GeomHeader), stream));
    auto mark = [](int i, cudaStream_t s) { prof_mark(true, i, s); };
    auto no_mark = [](int, cudaStream_t) {};
    prof_mark(true, 0, stream);
    if (a->P > 0) {
        // V views: every view is projected, depth-sorted and binned on its own (the binning appends its lists behind the
        // previous view's in the one binning buffer); the compositors then run once over the tall grid of all views.
        // The stage marks of the front end are those of the last view: the earlier views' binning counts as projection.
        for (int v = 0; v < V; ++v) {
            const RasterBuffers s = view_slice(b, v);
            const bool last = v == V - 1;
            if ((rc = launch_projection(*a, s, v, stream)) != 0) return rc;
            if (last) prof_mark(true, 1, stream);
            if ((rc = launch_binning(a->P, s, num_sms(), stream, last ? (stage_mark_fn)mark : (stage_mark_fn)no_mark,
                                     a->num_rendered_host ? a->num_rendered_host + v : nullptr,
                                     last ? a->count_ready_event : nullptr)) != 0) return rc;
        }
        if (V > 1 && (rc = launch_tile_order(b, stream)) != 0) return rc;
        g_launches += V * (1 + (1 + R3DG_SORT_MAX_PASSES) + 4) + (V > 1 ? 1 : 0);   // per view: project; histogram + radix passes; count, colsum + starts, apply, scatter; tile order
    } else {
        if ((rc = launch_empty_binning(b, stream)) != 0) return rc;
        for (int i = 1; i <= 4; ++i) prof_mark(true, i, stream);
        g_launches += 1;                                    // starts (empty ranges, tile order)
    }
    prof_mark(true, 5, stream);
    if ((rc = launch_composite_forward(*a, b, stream, mark)) != 0) return rc;
    prof_mark(true, 7, stream);
    g_launches += 1 + (a->computer_pseudo_normal ? V : 0) + (a->deterministic && a->P > 0 ? 1 : 0);   // composite, normals, weights
    if (g_prof.on) g_prof.fwd_calls++;
    if (a->P == 0) {      // (P > 0: the counts were written, and the event recorded, as soon as the binning offsets existed)
        for (int v = 0; v < V && a->num_rendered_host; ++v)
            R3DG_CUDA_TRY(cudaMemcpyAsync(a->num_rendered_host + v, b.header + v, sizeof(int), cudaMemcpyDeviceToHost, stream));
        if (a->count_ready_event) R3DG_CUDA_TRY(cudaEventRecord((cudaEvent_t)a->count_ready_event, stream));
    }
    if (a->debug) {   // reference CHECK_CUDA semantics (auxiliary.h:166-173): sync and report
        cudaError_t e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) return -(int)e;
    }
    return 0;
}

int r3dg_raster_backward(const r3dg_raster_bwd_args* a, r3dg_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!a || a->P < 0 || a->W <= 0 || a->H <= 0 || a->S < 0) return R3DG_ERR_BAD_ARG;
    if (a->S > R3DG_MAX_S_BWD) return R3DG_ERR_UNSUPPORTED;
    const int V = views_of(a->V, a->view_cams, a->P);
    if (V == 0) return R3DG_ERR_BAD_ARG;
    if (misaligned16(a->rotations) || misaligned16(a->dL_drotations)) return R3DG_ERR_BAD_ARG;
    // ray-depth mode: the gradient rows are one float4 wider
    const size_t det_rows_bytes = a->ray_depth ? r3dg_raster_ray_depth_bwd_det_bytes(V * a->P, a->S) : r3dg_raster_bwd_det_bytes(V * a->P, a->S);
    if (a->deterministic && (!a->det_work || a->det_work_bytes < det_rows_bytes)) return R3DG_ERR_BAD_ARG;
    const int cam_outs = (a->dL_dviewmatrix != nullptr) + (a->dL_dprojmatrix != nullptr) + (a->dL_dcampos != nullptr);
    // appearance-only mode: every geometry output NULL (the six per-Gaussian ones and the camera gradients).  P = 0
    // writes no per-Gaussian output, and is refused for none of them, as before this mode existed.
    const int geo_outs = (a->dL_dmeans2D != nullptr) + (a->dL_dopacity != nullptr) + (a->dL_dmeans3D != nullptr) +
                         (a->dL_dcov3D != nullptr) + (a->dL_dscales != nullptr) + (a->dL_drotations != nullptr);
    const bool geometry = geo_outs == 6 || a->P == 0;
    if (a->P > 0 && geo_outs != 0 && geo_outs != 6) return R3DG_ERR_BAD_ARG;
    // absgrad: the deterministic workspace grows only when it is requested (the appearance-only mode ignores it)
    if (a->deterministic && geometry && a->dL_dmeans2D_abs &&
        a->det_work_bytes < det_rows_bytes + r3dg_raster_bwd_det_absgrad_bytes(V * a->P)) return R3DG_ERR_BAD_ARG;
    if (!geometry && (cam_outs != 0 || (!a->dL_dcolors && !a->dL_dfeatures && !a->dL_dsh))) return R3DG_ERR_BAD_ARG;
    if (V > 1 && a->P > 0 && a->shs && (geometry || a->dL_dsh) && (!a->dL_dsh_factor || !a->dL_dsh)) return R3DG_ERR_BAD_ARG;
    if (cam_outs != 0 && cam_outs != 3) return R3DG_ERR_BAD_ARG;
    if (geometry && a->filter_3d && (a->cov3D_precomp || !a->opacities)) return R3DG_ERR_BAD_ARG;
    // depth statistics: the flag with both cotangents and the forward's larger image buffer, or neither cotangent
    const bool ds = geometry && a->depth_stats != 0;
    if (ds && (!a->dL_dout_depth2 || !a->dL_dout_median_depth ||
               a->img_bytes < r3dg_raster_depth_stats_img_bytes(a->W, a->H, V))) return R3DG_ERR_BAD_ARG;
    if (geometry && !ds && (a->dL_dout_depth2 || a->dL_dout_median_depth)) return R3DG_ERR_BAD_ARG;
    const bool cam = cam_outs == 3;
    if (cam && (!a->cam_work || a->cam_work_bytes < r3dg_raster_cam_grad_bytes(a->P, V))) return R3DG_ERR_BAD_ARG;
    // (appearance-only: the opacity, depth, pseudo-normal and surface-xyz cotangents have no appearance gradient)
    const bool surface = geometry && (a->dL_dout_normal || a->dL_dout_surface_xyz);
    if (surface && (!a->fwd_opacity || !a->fwd_depth || !a->dL_dout_opacity || !a->dL_dout_depth || !a->surface_work ||
                    a->surface_work_bytes < r3dg_raster_surface_grad_bytes(a->W, a->H, V))) return R3DG_ERR_BAD_ARG;
    if (a->P == 0) {
        if (cam) {
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dviewmatrix, 0, (size_t)V * 16 * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dprojmatrix, 0, (size_t)V * 16 * sizeof(float), stream));
            R3DG_CUDA_TRY(cudaMemsetAsync(a->dL_dcampos, 0, (size_t)V * 3 * sizeof(float), stream));
        }
        return 0;
    }
    RasterBuffers b;
    int rc = raster_buffers(a->P, a->S, a->W, a->H, a->geom, a->geom_bytes, a->img, a->img_bytes, a->binning,
                            a->binning_bytes, b, V, a->ray_depth != 0, ds);
    if (rc != 0) return rc;
    prof_mark(false, 8, stream);
    // pseudo-normal / surface-xyz cotangents: their pull-back joins the depth and opacity cotangents, and the compositor
    // runs on the sums (its stage of the profiler includes this pass)
    r3dg_raster_bwd_args sa;
    const bool surface_cam = surface && cam && a->dL_dout_normal;
    const int surface_blocks = surface_grad_blocks(a->W, a->H);
    float* surface_part = nullptr;
    if (surface) {
        float* planes = (float*)a->surface_work;
        surface_part = surface_cam ? (float*)((char*)a->surface_work + align_up(2 * (size_t)V * a->W * a->H * sizeof(float), 256))
                                   : nullptr;
        if ((rc = launch_surface_backward(*a, V, planes, surface_part, stream)) != 0) return rc;
        sa = *a;
        sa.dL_dout_depth = planes;
        sa.dL_dout_opacity = planes + (size_t)V * a->W * a->H;
        a = &sa;
    }
    if ((rc = launch_composite_backward(*a, b, geometry, stream)) != 0) return rc;
    prof_mark(false, 9, stream);
    // one projection backward per view, in view order: view 0 writes the summed gradients, every later view adds its
    // own to them (a left fold in fp32), per-view outputs go to the view's rows.  Appearance-only: one launch for all
    // views writes the colour, feature and SH outputs the same way (the profiler counts it as the projection backward).
    if (geometry) {
        for (int v = 0; v < V; ++v)
            if ((rc = launch_projection_backward(*a, view_slice(b, v), v, stream)) != 0) return rc;
    } else if ((rc = launch_appearance_backward(*a, b, stream)) != 0) {
        return rc;
    }
    if (V > 1 && a->shs && a->dL_dsh) {     // dL_dsh from the views' rank-1 factors, views in order
        if ((rc = r3dg_sh_grad_from_factors(a->P, a->D, a->M, V, a->means3D, a->campos, a->dL_dsh_factor, 1.0f, a->dL_dsh,
                                            stream_)) != 0) return rc;
    }
    if (cam) {                      // every view's camera gradients from its CTAs' partial sums
        const CamGradOut o = {{a->dL_dviewmatrix, a->dL_dprojmatrix, a->dL_dcampos}, {16, 16, 3}};
        if ((rc = launch_cam_grad_sum((const float*)a->cam_work, cam_grad_blocks(a->P), V, o, stream)) != 0) return rc;
    }
    if (surface_cam &&              // then the pseudo-normal's term of dL/dviewmatrix, added after the projection's
        (rc = launch_surface_cam_sum(surface_part, surface_blocks, V, a->dL_dviewmatrix, stream)) != 0) return rc;
    prof_mark(false, 10, stream);
    // zeroing of the composited rows (deterministic mode: and the cotangent scale), CTA order, composite, projection per view (appearance-only: one launch), camera
    // sums (the SH rebuild counts itself); surface pass per view and its camera sums
    g_launches += 3 + (geometry ? V : 1) + (cam ? 1 : 0) + (surface ? V : 0) + (surface_cam ? 1 : 0);
    if (g_prof.on) g_prof.bwd_calls++;
    if (a->debug) {
        cudaError_t e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) return -(int)e;
    }
    return 0;
}

extern unsigned long long r3dg_adam_launches, r3dg_shx_launches;
unsigned long long r3dg_launch_count(void) { return g_launches + r3dg_adam_launches + r3dg_shx_launches; }

int r3dg_tune(const char* key, int value, int* previous) {
    if (!key) return R3DG_ERR_BAD_ARG;
    int prev = 0;
    int rc = shade_tune(key, value, &prev);                       // each returns R3DG_ERR_UNSUPPORTED for a key it does not own
    if (rc == R3DG_ERR_UNSUPPORTED) rc = composite_tune(key, value, &prev);
    if (rc == R3DG_ERR_UNSUPPORTED) rc = composite_bwd_tune(key, value, &prev);
    if (previous) *previous = prev;
    return rc;
}

int r3dg_prof_begin(int max_calls) {
    for (auto& e : g_prof.ev) cudaEventDestroy(e);
    g_prof.ev.assign((size_t)max_calls * (ST_COUNT + 2), nullptr);
    for (auto& e : g_prof.ev) R3DG_CUDA_TRY(cudaEventCreate(&e));
    g_prof.max_calls = max_calls; g_prof.fwd_calls = g_prof.bwd_calls = 0; g_prof.on = true;
    return 0;
}

// Sums the per-stage durations (ms) over the recorded calls; the caller must have synchronised.
int r3dg_prof_end(float* stage_ms /*[9]*/, int* fwd_calls, int* bwd_calls) {
    g_prof.on = false;
    for (int i = 0; i < ST_COUNT; ++i) stage_ms[i] = 0.f;
    const int nf = g_prof.fwd_calls < g_prof.max_calls ? g_prof.fwd_calls : g_prof.max_calls;
    const int nb = g_prof.bwd_calls < g_prof.max_calls ? g_prof.bwd_calls : g_prof.max_calls;
    for (int c = 0; c < nf; ++c)
        for (int i = 0; i < 7; ++i) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, g_prof.at(c, i), g_prof.at(c, i + 1)) == cudaSuccess) stage_ms[i] += ms;
        }
    for (int c = 0; c < nb; ++c)
        for (int i = 0; i < 2; ++i) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, g_prof.at(c, 8 + i), g_prof.at(c, 9 + i)) == cudaSuccess) stage_ms[7 + i] += ms;
        }
    if (fwd_calls) *fwd_calls = nf;
    if (bwd_calls) *bwd_calls = nb;
    for (auto& e : g_prof.ev) cudaEventDestroy(e);
    g_prof.ev.clear();
    return 0;
}

int r3dg_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                      uint8_t* present, r3dg_stream_t stream) {
    (void)projmatrix;   // the reference's in_frustum computes p_proj but never uses it (auxiliary.h:151-154)
    g_launches += P > 0 ? 1 : 0;
    return launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream);
}

// ---- BVH visibility (bvh_tracing._C) -------------------------------------------------------
size_t r3dg_bvh_build_tmp_bytes(int P) { return bvh_build_tmp_bytes(P); }
size_t r3dg_bvh_trace_tmp_bytes(int P) { return bvh_packets_bytes(P); }

int r3dg_bvh_leaf_aabbs(int P, const float* means3D, const float* scales, const float* rotations,
                        int32_t* nodes, float* aabbs, r3dg_stream_t stream) {
    if (misaligned16(rotations)) return R3DG_ERR_BAD_ARG;
    g_launches += P > 0 ? 1 : 0;
    return launch_bvh_leaf_aabbs(P, means3D, scales, rotations, nodes, aabbs, (cudaStream_t)stream);
}

int r3dg_bvh_build(int P, int32_t* nodes, float* aabbs, uint64_t* morton, void* tmp, size_t tmp_bytes,
                   r3dg_stream_t stream) {
    if (P < 0) return R3DG_ERR_BAD_ARG;
    g_launches += P > 0 ? 6 + 1 + R3DG_SORT_MAX_PASSES : 0;
    return launch_bvh_build(P, nodes, aabbs, morton, tmp, tmp_bytes, num_sms(), (cudaStream_t)stream);
}

int r3dg_bvh_trace_opacity(int P, long long num_rays, const int32_t* nodes, const float* aabbs,
                           const float* rays_o, int rays_per_origin, float origin_offset, const float* rays_d,
                           const float* means3D, const float* covs3D, const float* opacities,
                           const float* normals, int32_t* num_contributes, float* rendered_opacity,
                           void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    if (P < 0 || num_rays < 0) return R3DG_ERR_BAD_ARG;
    g_launches += (P > 0 && num_rays > 0) ? 2 : 0;
    return launch_bvh_trace(P, num_rays, nodes, aabbs, rays_o, rays_per_origin, origin_offset, rays_d, means3D, covs3D,
                            opacities, normals, num_contributes, rendered_opacity, tmp, tmp_bytes, num_sms(),
                            (cudaStream_t)stream);
}

int r3dg_sample_incident_dirs(int P, int N, const float* normals, const float* phase, float* dirs, float* areas, r3dg_stream_t stream) {
    if (P < 0 || N < 0) return R3DG_ERR_BAD_ARG;
    g_launches += (P > 0 && N > 0) ? 1 : 0;
    return launch_sample_dirs(P, N, normals, phase, dirs, areas, num_sms(), (cudaStream_t)stream);
}

int r3dg_bvh_bake_visibility(int P, int first_slot, int count, int N, const int32_t* nodes, const float* aabbs,
                             const float* means3D, const float* covs3D, const float* opacities, const float* normals,
                             float origin_offset, int32_t* num_contributes, float* visibility, float* dirs, float* areas,
                             void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    if (P < 0 || count < 0 || N < 0) return R3DG_ERR_BAD_ARG;
    g_launches += (P > 0 && count > 0 && N > 0) ? 2 : 0;
    return launch_bvh_bake(P, first_slot, count, N, nodes, aabbs, means3D, covs3D, opacities, normals, origin_offset,
                           num_contributes, visibility, dirs, areas, tmp, tmp_bytes, num_sms(), (cudaStream_t)stream);
}

// ---- ray-traced indirect light ------------------------------------------------------------
size_t r3dg_bvh_bake_radiance_tmp_bytes(int P) { return bvh_radiance_tmp_bytes(P); }

int r3dg_bvh_bake_radiance(int P, int N, const int32_t* nodes, const float* aabbs, const float* means3D,
                           const float* covs3D, const float* opacities, const float* normals, const float* shs, int M,
                           int sh_degree, float origin_offset, float* radiance, float* transmittance, int32_t* num_hits,
                           void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    const int rc = launch_bvh_radiance(P, N, nodes, aabbs, means3D, covs3D, opacities, normals, shs, M, sh_degree, origin_offset,
                                       radiance, transmittance, num_hits, tmp, tmp_bytes, (cudaStream_t)stream);
    g_launches += (rc == 0 && P > 0 && N > 0) ? 2 : 0;
    return rc;
}

int r3dg_fit_incident_sh(int P, int N, const float* radiance, const float* normals, int degree, float ridge, float* out,
                         r3dg_stream_t stream) {
    const int rc = launch_fit_incident_sh(P, N, radiance, normals, degree, ridge, out, (cudaStream_t)stream);
    g_launches += (rc == 0 && P > 0) ? 1 : 0;
    return rc;
}

// ---- point and directional lights (lights.py) -----------------------------------------------
size_t r3dg_bvh_trace_lights_tmp_bytes(int P) { return bvh_lights_tmp_bytes(P); }

int r3dg_bvh_trace_lights(int P, int K, const int32_t* kind, const float* vec, const int32_t* nodes, const float* aabbs,
                          const float* means3D, const float* covs3D, const float* opacities, const float* normals,
                          float* shadows, void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_bvh_lights(P, K, kind, vec, nodes, aabbs, means3D, covs3D, opacities, normals, shadows, tmp, tmp_bytes,
                                     num_sms(), (cudaStream_t)stream, &launched);
    g_launches += launched ? 2 : 0;                       // pack, trace
    return rc;
}

size_t r3dg_shade_lights_work_bytes(int P, int K) { return shade_lights_work_bytes(P, K); }

int r3dg_shade_lights_forward(const r3dg_light_args* args, r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_shade_lights_forward(args, (cudaStream_t)stream, &launched);
    g_launches += launched ? 1 : 0;
    return rc;
}

int r3dg_shade_lights_backward(const r3dg_light_args* args, r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_shade_lights_backward(args, (cudaStream_t)stream, &launched);
    g_launches += launched ? 2 : 0;                       // Gaussians, fixed-order light reduction
    return rc;
}

// ---- spot and rect lights (lights.py, ShapedLights) ---------------------------------------------
int r3dg_shaped_lights_num_rays(int K, const int32_t* kind, int M) { return shaped_num_rays(K, kind, M); }

size_t r3dg_bvh_trace_shaped_lights_tmp_bytes(int P) { return bvh_lights_tmp_bytes(P); }

int r3dg_bvh_trace_shaped_lights(const r3dg_shaped_light_args* args, const int32_t* nodes, const float* aabbs,
                                 const float* covs3D, const float* opacities, float* shadows, void* tmp, size_t tmp_bytes,
                                 r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_bvh_shaped_lights(args, nodes, aabbs, covs3D, opacities, shadows, tmp, tmp_bytes, num_sms(),
                                            (cudaStream_t)stream, &launched);
    g_launches += launched ? 2 : 0;                       // pack, trace
    return rc;
}

size_t r3dg_shade_shaped_lights_work_bytes(int P, int K) { return shade_shaped_lights_work_bytes(P, K); }

int r3dg_shade_shaped_lights_forward(const r3dg_shaped_light_args* args, r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_shade_shaped_lights_forward(args, (cudaStream_t)stream, &launched);
    g_launches += launched ? 1 : 0;
    return rc;
}

int r3dg_shade_shaped_lights_backward(const r3dg_shaped_light_args* args, r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_shade_shaped_lights_backward(args, (cudaStream_t)stream, &launched);
    g_launches += launched ? 2 : 0;                       // Gaussians, per-light reduction
    return rc;
}

// ---- similarity transforms of Gaussian models (compose.py) --------------------------------------
size_t r3dg_compose_work_bytes(int P, int K) { return compose_work_bytes(P, K); }

int r3dg_compose_forward(const r3dg_compose_args* args, r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_compose_forward(args, (cudaStream_t)stream, &launched);
    g_launches += launched ? 1 : 0;
    return rc;
}

int r3dg_compose_backward(const r3dg_compose_args* args, r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_compose_backward(args, (cudaStream_t)stream, &launched);
    g_launches += launched ? 2 : 0;                       // rows, fixed-order pose reduction
    return rc;
}

int r3dg_unpremultiply_forward(int S, long long HW, const float* feature, const float* opacity, const int32_t* n_contrib,
                               float* out, r3dg_stream_t stream) {
    if (S < 0 || HW < 0) return R3DG_ERR_BAD_ARG;
    g_launches += (S > 0 && HW > 0) ? 1 : 0;
    return launch_unpremultiply_forward(S, HW, feature, opacity, n_contrib, out, num_sms(), (cudaStream_t)stream);
}
int r3dg_unpremultiply_backward(int S, long long HW, const float* feature, const float* opacity, const int32_t* n_contrib,
                                const float* dL_dout, float* dL_dfeature, float* dL_dopacity, r3dg_stream_t stream) {
    if (S < 0 || HW < 0) return R3DG_ERR_BAD_ARG;
    g_launches += HW > 0 ? 1 : 0;
    return launch_unpremultiply_backward(S, HW, feature, opacity, n_contrib, dL_dout, dL_dfeature, dL_dopacity, num_sms(), (cudaStream_t)stream);
}

int r3dg_pack_features_forward(int P, int S, const float* means3D, const float* viewmatrix, int num, const r3dg_pack_src* srcs,
                               float* out, r3dg_stream_t stream) {
    if (num > 0 && !srcs) return R3DG_ERR_BAD_ARG;
    g_launches += P > 0 ? 1 : 0;
    return launch_pack_features_forward(P, S, means3D, viewmatrix, num, srcs, out, num_sms(), (cudaStream_t)stream);
}
int r3dg_pack_features_backward(int P, int S, const float* means3D, const float* viewmatrix, const float* dL_dout, int num,
                                const r3dg_pack_src* dsts, float* dL_dmeans3D, float* dL_dviewmatrix, void* work,
                                size_t work_bytes, r3dg_stream_t stream) {
    if (num > 0 && !dsts) return R3DG_ERR_BAD_ARG;
    g_launches += P > 0 ? (dL_dviewmatrix ? 3 : 1) : 0;
    return launch_pack_features_backward(P, S, means3D, viewmatrix, dL_dout, num, dsts, dL_dmeans3D, dL_dviewmatrix, work,
                                         work_bytes, num_sms(), (cudaStream_t)stream);
}

size_t r3dg_compact_tmp_bytes(int P) { return compact_tmp_bytes(P < 0 ? 0 : P); }
int r3dg_compact_scan(int P, const uint8_t* keep, void* tmp, size_t tmp_bytes, int* count_host, r3dg_stream_t stream) {
    if (P < 0 || !tmp) return R3DG_ERR_BAD_ARG;
    g_launches += P > 0 ? 3 : 1;
    return launch_compact_scan(P, keep, tmp, tmp_bytes, count_host, (cudaStream_t)stream);
}
int r3dg_compact_rows(int P, int num_tensors, const r3dg_compact_tensor* tensors, const uint8_t* keep, const void* tmp,
                      r3dg_stream_t stream) {
    if (P < 0 || num_tensors < 0 || (num_tensors > 0 && !tensors)) return R3DG_ERR_BAD_ARG;
    g_launches += (P > 0 && num_tensors > 0) ? (num_tensors + R3DG_COMPACT_MAX - 1) / R3DG_COMPACT_MAX : 0;
    return launch_compact_rows(P, num_tensors, tensors, keep, tmp, num_sms(), (cudaStream_t)stream);
}

// ---- GaussianModel.add_densification_stats / densify_and_prune ------------------------------------
int r3dg_densify_stats(int P, const float* viewspace_grad, int grad_stride, const float* normal_grad,
                       const uint8_t* update_filter, const float* weights, const int32_t* radii, float* weights_accum,
                       float* xyz_gradient_accum, float* normal_gradient_accum, float* denom, float* max_radii2D,
                       r3dg_stream_t stream) {
    const int rc = launch_densify_stats(P, viewspace_grad, grad_stride, normal_grad, update_filter, weights, radii, weights_accum,
                                        xyz_gradient_accum, normal_gradient_accum, denom, max_radii2D, (cudaStream_t)stream);
    if (rc == 0 && P > 0) g_launches += 1;
    return rc;
}
size_t r3dg_densify_tmp_bytes(int P) { return densify_tmp_bytes(P < 0 ? 0 : P); }
int r3dg_densify_classify(int P, const float* xyz_gradient_accum, const float* normal_gradient_accum, const float* denom,
                          const float* weights_accum, const float* scaling, const float* opacity,
                          const r3dg_densify_thresholds* thresholds, void* tmp, size_t tmp_bytes, int* totals_host,
                          r3dg_stream_t stream) {
    if (!thresholds) return R3DG_ERR_BAD_ARG;
    const int rc = launch_densify_classify(P, xyz_gradient_accum, normal_gradient_accum, denom, weights_accum, scaling, opacity,
                                           *thresholds, tmp, tmp_bytes, totals_host, (cudaStream_t)stream);
    if (rc == 0) g_launches += P > 0 ? 3 : 1;     // classify, scan, offsets
    return rc;
}
int r3dg_densify_apply(int P, const int* totals, int num_tensors, const r3dg_densify_tensor* tensors, const float* rotation,
                       const float* scaling, const float* samples, float split_recip, const void* tmp, size_t tmp_bytes,
                       r3dg_stream_t stream) {
    if (misaligned16(rotation)) return R3DG_ERR_BAD_ARG;
    const int rc = launch_densify_apply(P, totals, num_tensors, tensors, rotation, scaling, samples, split_recip, tmp, tmp_bytes,
                                        num_sms(), (cudaStream_t)stream);
    if (rc == 0 && P > 0 && num_tensors > 0) g_launches += 1;
    return rc;
}

// ---- MCMC densification (mcmc.py) ----------------------------------------------------------------
size_t r3dg_mcmc_tmp_bytes(int P, int n_new) { return mcmc_tmp_bytes(P < 0 ? 0 : P, n_new < 0 ? 0 : n_new); }
int r3dg_mcmc_noise(int P, float* xyz, const float* rotation, const float* scaling, const float* opacity, const float* z,
                    double scale, double k, double t, r3dg_stream_t stream) {
    const int rc = launch_mcmc_noise(P, xyz, rotation, scaling, opacity, z, scale, k, t, (cudaStream_t)stream);
    if (rc == 0 && P > 0) g_launches += 1;
    return rc;
}
int r3dg_mcmc_classify(int P, const float* opacity, float min_opacity, void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    const int rc = launch_mcmc_classify(P, opacity, min_opacity, tmp, tmp_bytes, (cudaStream_t)stream);
    if (rc == 0) g_launches += 3;        // classify, block-sum scan, cdf
    return rc;
}
int r3dg_mcmc_apply(int P, int n_new, const float* uniforms, const float* opacity, const float* scaling, double min_opacity,
                    int n_max, int num_tensors, const r3dg_densify_tensor* tensors, void* tmp, size_t tmp_bytes,
                    r3dg_stream_t stream) {
    const int rc = launch_mcmc_apply(P, n_new, uniforms, opacity, scaling, min_opacity, n_max, num_tensors, tensors, tmp,
                                     tmp_bytes, num_sms(), (cudaStream_t)stream);
    if (rc == 0) g_launches += 3;        // draw, source update, apply
    return rc;
}

// ---- Mip-Splatting's 3D filter (filter3d.py) -------------------------------------------------------
size_t r3dg_filter3d_tmp_bytes(int P) { return filter3d_tmp_bytes(P < 0 ? 0 : P); }
int r3dg_filter3d_compute(int P, int V, const float* means3D, const float* viewmatrices, const float* intrinsics,
                          float focal_max, float* filter_3d, void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    const int rc = launch_filter3d(P, V, means3D, viewmatrices, intrinsics, focal_max, filter_3d, tmp, tmp_bytes, num_sms(),
                                   (cudaStream_t)stream);
    if (rc == 0 && P > 0) g_launches += 2;        // least valid depth, finish
    return rc;
}

// ---- simple_knn._C.distCUDA2 ----------------------------------------------------------------
size_t r3dg_knn_tmp_bytes(int P) { return knn_tmp_bytes(P); }
int r3dg_knn_dist2(int P, const float* points, float* mean_dist2, void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    if (P < 0) return R3DG_ERR_BAD_ARG;
    g_launches += P > 0 ? 6 + 1 + R3DG_SORT_MAX_PASSES : 0;
    return launch_knn(P, points, mean_dist2, tmp, tmp_bytes, num_sms(), (cudaStream_t)stream);
}

// ---- utils.loss_utils.ssim ----------------------------------------------------------------------
size_t r3dg_ssim_tmp_bytes(int N, int C, int H, int W) { return ssim_tmp_bytes(N, C, H, W); }
int r3dg_ssim_forward(int N, int C, int H, int W, const float* img1, const float* img2, int size_average, float* out,
                      void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    const int rc = launch_ssim_forward(N, C, H, W, img1, img2, size_average, out, tmp, tmp_bytes, (cudaStream_t)stream);
    if (rc == 0) g_launches += 2;        // tiles, reduction
    return rc;
}
int r3dg_ssim_backward(int N, int C, int H, int W, const float* img1, const float* img2, int size_average,
                       const float* dL_dout, float* dL_dimg1, r3dg_stream_t stream) {
    const int rc = launch_ssim_backward(N, C, H, W, img1, img2, size_average, dL_dout, dL_dimg1, (cudaStream_t)stream);
    if (rc == 0) g_launches += 1;
    return rc;
}

// ---- utils.loss_utils.first_order_edge_aware_loss / tv_loss ---------------------------------------
size_t r3dg_edge_aware_tmp_bytes(int Cd, int Ci, int H, int W) { return edge_aware_tmp_bytes(Cd, Ci, H, W); }
int r3dg_edge_aware_forward(int Cd, int Ci, int H, int W, const float* data, const float* img, float* out, void* tmp,
                            size_t tmp_bytes, r3dg_stream_t stream) {
    const int rc = launch_edge_aware_forward(Cd, Ci, H, W, data, img, out, tmp, tmp_bytes, (cudaStream_t)stream);
    if (rc == 0) g_launches += 2;        // tiles, reduction
    return rc;
}
int r3dg_edge_aware_backward(int Cd, int Ci, int H, int W, const float* data, const float* img, const float* dL_dout,
                             float* dL_ddata, float* dL_dimg, r3dg_stream_t stream) {
    const int rc = launch_edge_aware_backward(Cd, Ci, H, W, data, img, dL_dout, dL_ddata, dL_dimg, (cudaStream_t)stream);
    if (rc == 0) g_launches += 1;
    return rc;
}
size_t r3dg_tv_tmp_bytes(int B, int H, int W) { return tv_tmp_bytes(B, H, W); }
int r3dg_tv_forward(int B, int H, int W, const float* x, float* out, void* tmp, size_t tmp_bytes, r3dg_stream_t stream) {
    const int rc = launch_tv_forward(B, H, W, x, out, tmp, tmp_bytes, (cudaStream_t)stream);
    if (rc == 0) g_launches += 2;        // blocks, reduction
    return rc;
}
int r3dg_tv_backward(int B, int H, int W, const float* x, const float* dL_dout, float* dL_dx, r3dg_stream_t stream) {
    const int rc = launch_tv_backward(B, H, W, x, dL_dout, dL_dx, (cudaStream_t)stream);
    if (rc == 0) g_launches += 1;
    return rc;
}

// ---- bilateral-grid colour correction (bilagrid.py) ------------------------------------------------
size_t r3dg_bilagrid_tmp_bytes(int G, int N, int H, int W, int GX, int GY, int L) {
    return bilagrid_tmp_bytes(G, N, H, W, GX, GY, L);
}
int r3dg_bilagrid_forward(int G, int N, int H, int W, int GX, int GY, int L, const float* grids, const int* image_ids,
                          const float* rgb, float* out, r3dg_stream_t stream) {
    const int rc = launch_bilagrid_forward(G, N, H, W, GX, GY, L, grids, image_ids, rgb, out, (cudaStream_t)stream);
    if (rc == 0) g_launches += 1;
    return rc;
}
int r3dg_bilagrid_backward(int G, int N, int H, int W, int GX, int GY, int L, const float* grids, const int* image_ids,
                           const float* rgb, const float* dL_dout, float* dL_drgb, float* dL_dgrids, void* tmp,
                           size_t tmp_bytes, r3dg_stream_t stream) {
    const int rc = launch_bilagrid_backward(G, N, H, W, GX, GY, L, grids, image_ids, rgb, dL_dout, dL_drgb, dL_dgrids, tmp,
                                            tmp_bytes, (cudaStream_t)stream);
    if (rc == 0) g_launches += dL_dgrids ? 2 : 1;        // tiles (+ partial reduction)
    return rc;
}

// ---- multi-view consistency losses (multiview.py) -------------------------------------------------
size_t r3dg_multiview_work_bytes(int B, int H, int W) { return multiview_work_bytes(B, H, W); }
size_t r3dg_multiview_det_bytes(int V, int H, int W) { return multiview_det_bytes(V, H, W); }
int r3dg_multiview_forward(const r3dg_multiview_args* args, r3dg_stream_t stream) {
    const int rc = launch_multiview_forward(args, (cudaStream_t)stream);
    if (rc == 0) g_launches += 2;                         // pixels, fixed-order reduction
    return rc;
}
int r3dg_multiview_backward(const r3dg_multiview_args* args, r3dg_stream_t stream) {
    const int rc = launch_multiview_backward(args, (cudaStream_t)stream);
    if (rc == 0) g_launches += args->deterministic ? 2 : 1;   // pixels (+ fixed-point read-back)
    return rc;
}

// ---- TSDF fusion and marching cubes (tsdf.py) -----------------------------------------------------
size_t r3dg_tsdf_extract_work_bytes(int NX, int NY, int NZ) { return tsdf_extract_work_bytes(NX, NY, NZ); }
int r3dg_tsdf_integrate(const r3dg_tsdf_integrate_args* args, r3dg_stream_t stream) {
    const int rc = launch_tsdf_integrate(args, (cudaStream_t)stream);
    if (rc == 0) g_launches += 1;
    return rc;
}
int r3dg_tsdf_extract_count(const r3dg_tsdf_extract_args* args, r3dg_stream_t stream) {
    bool launched = false;
    const int rc = launch_tsdf_extract_count(args, (cudaStream_t)stream, &launched);
    if (launched) g_launches += 2;                        // classify, scan
    return rc;
}
int r3dg_tsdf_extract_emit(const r3dg_tsdf_extract_args* args, r3dg_stream_t stream) {
    const int rc = launch_tsdf_extract_emit(args, (cudaStream_t)stream);
    if (rc == 0 && (args->n_verts > 0 || args->n_faces > 0)) g_launches += 2;   // vertices, faces
    return rc;
}

namespace {
__global__ void unpack_rec_kernel(int P, int recf, int what, const float* __restrict__ rec,
                                  const uint32_t* __restrict__ tiles, float* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const bool vis = tiles[i] > 0;
    const float* r = rec + (size_t)i * recf;
    switch (what) {
        case 0: dst[i] = vis ? r[6] : 0.f; break;                                   // depths
        case 3: dst[2 * i] = vis ? r[0] : 0.f; dst[2 * i + 1] = vis ? r[1] : 0.f; break;
        case 5: dst[4 * i] = vis ? r[2] : 0.f; dst[4 * i + 1] = vis ? r[3] : 0.f;
                dst[4 * i + 2] = vis ? r[4] : 0.f; dst[4 * i + 3] = vis ? r[5] : 0.f; break;
        case 6: dst[3 * i] = vis ? r[8] : 0.f; dst[3 * i + 1] = vis ? r[9] : 0.f; dst[3 * i + 2] = vis ? r[10] : 0.f; break;
    }
}
__global__ void unpack_clamped_kernel(int P, const uint8_t* __restrict__ cl, const uint32_t* __restrict__ tiles,
                                      uint8_t* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const unsigned c = tiles[i] > 0 ? cl[i] : 0u;
    dst[3 * i] = c & 1u; dst[3 * i + 1] = (c >> 1) & 1u; dst[3 * i + 2] = (c >> 2) & 1u;
}
__global__ void unpack_composited_kernel(int P, const uint8_t* __restrict__ cl, uint8_t* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < P) dst[i] = (cl[i] & kComposited) ? 1 : 0;
}
}  // namespace

static long long debug_copy(bool ray_depth, int id, int P, int S, int W, int H, const void* geom_, const void* img_,
                            const void* bin_, size_t binning_bytes, void* dst, long long max_bytes,
                            r3dg_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    RasterBuffers b;       // the geom and img sizes are not given: only the binning buffer's is checked
    const bool binned = raster_buffers(P, S, W, H, const_cast<void*>(geom_), SIZE_MAX, const_cast<void*>(img_), SIZE_MAX,
                                       const_cast<void*>(bin_), binning_bytes, b, 1, ray_depth) == 0;
    const size_t HW = (size_t)W * H;
    const float* rec = b.rec;
    const uint32_t* tt = b.tiles_touched;
    const int nb = (P + 255) / 256;
    auto copy = [&](const void* src, size_t n) -> long long {
        if ((long long)n > max_bytes) n = (size_t)max_bytes;
        if (cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, stream) != cudaSuccess) return -2;
        return (long long)n;
    };
    switch (id) {
        case 0: if (max_bytes < 4LL * P) return -1; if (P) unpack_rec_kernel<<<nb, 256, 0, stream>>>(P, b.recf, 0, rec, tt, (float*)dst); return 4LL * P;
        case 1: if (max_bytes < 3LL * P) return -1; if (P) unpack_clamped_kernel<<<nb, 256, 0, stream>>>(P, b.clamped, tt, (uint8_t*)dst); return 3LL * P;
        case 3: if (max_bytes < 8LL * P) return -1; if (P) unpack_rec_kernel<<<nb, 256, 0, stream>>>(P, b.recf, 3, rec, tt, (float*)dst); return 8LL * P;
        case 5: if (max_bytes < 16LL * P) return -1; if (P) unpack_rec_kernel<<<nb, 256, 0, stream>>>(P, b.recf, 5, rec, tt, (float*)dst); return 16LL * P;
        case 6: if (max_bytes < 12LL * P) return -1; if (P) unpack_rec_kernel<<<nb, 256, 0, stream>>>(P, b.recf, 6, rec, tt, (float*)dst); return 12LL * P;
        case 7: return copy(tt, 4 * (size_t)P);
        case 8: {   // reference geomState.point_offsets: rebuilt on demand (not needed by the hot path)
            if (max_bytes < 4LL * P) return -1;
            if (P == 0) return 0;
            char* tmp = nullptr;
            const size_t state_bytes = ((size_t)P / R3DG_SCAN_ITEMS + 2) * 4;
            if (cudaMalloc(&tmp, 256 + state_bytes) != cudaSuccess) return -2;
            int rc = launch_point_offsets(P, tt, (uint32_t*)dst, (uint32_t*)(tmp + 256), (GeomHeader*)tmp, stream);
            cudaStreamSynchronize(stream);
            cudaFree(tmp);
            return rc == 0 ? 4LL * P : -2;
        }
        case 13: return copy(b.final_T, 4 * HW);
        case 14: return copy(b.n_contrib, 4 * HW);
        case 23: return copy(b.median_pos, 4 * HW);    // (the caller checks that the buffer has the region)
        case 15: return copy(b.ranges, 8 * (size_t)b.tiles);
        case 16: return copy(b.bwd_work, 8 * (size_t)b.tiles);
        case 17: return copy(b.bwd_order, 8 * (size_t)b.tiles);
        case 20: return copy(b.brects, 8 * (size_t)P);
        case 22: if (max_bytes < P) return -1; if (P) unpack_composited_kernel<<<nb, 256, 0, stream>>>(P, b.clamped, (uint8_t*)dst); return P;
        case 9: case 10: case 18: case 19: {
            if (!binned) return -1;
            // caller limits the copy to R entries through max_bytes
            if (id == 9) return copy(b.point_list, std::min((size_t)max_bytes, (size_t)b.capacity * 4));
            if (id == 18) return copy(b.bmask, std::min((size_t)max_bytes, (size_t)b.capacity));
            if (id == 19) return copy(b.cmask, std::min((size_t)max_bytes, (size_t)b.capacity));
            // reference binningState.point_list_keys (sorted): rebuilt from the lists
            const long long limit = std::min(max_bytes / 8, b.capacity);
            if (launch_rebuild_keys(b.tiles, b.ranges, b.point_list, rec, b.recf, limit, (uint64_t*)dst, stream) != 0) return -2;
            return limit * 8;
        }
    }
    return -1;
}

long long r3dg_raster_debug_copy(int id, int P, int S, int W, int H, const void* geom, const void* img,
                                 const void* binning, size_t binning_bytes, void* dst, long long max_bytes,
                                 r3dg_stream_t stream) {
    return debug_copy(false, id, P, S, W, H, geom, img, binning, binning_bytes, dst, max_bytes, stream);
}
long long r3dg_raster_ray_depth_debug_copy(int id, int P, int S, int W, int H, const void* geom, const void* img,
                                           const void* binning, size_t binning_bytes, void* dst, long long max_bytes,
                                           r3dg_stream_t stream) {
    return debug_copy(true, id, P, S, W, H, geom, img, binning, binning_bytes, dst, max_bytes, stream);
}

}  // extern "C"
