// Internal launcher declarations shared by the translation units of libr3dg_b200.so.
#pragma once
#include <cuda_runtime.h>
#include "../../include/r3dg_b200.h"
#include "common.cuh"
#include "detacc.cuh"

namespace r3dg {

// Typed views of the rasterizer's three caller-owned work buffers (regions described in api.cu, which alone knows
// their byte layout and fills and size-checks this once per call) and the values derived from the call's shapes.
struct RasterBuffers {
    GeomHeader* header;                                                            // geom: per Gaussian
    float *rec, *grad;
    uint32_t* tiles_touched;
    uint2 *rects, *brects;
    uint8_t* clamped;                                                              // bits 0-2: SH colour clamped; kComposited
    char* sort;                                                                    // laid out by sort_layout
    SortLayout sort_layout{0};
    float* final_T;                                                                // img: per pixel and per tile
    int* n_contrib;
    uint2* ranges;
    uint32_t *tile_order, *bwd_work, *bwd_order, *slab_sum, *bin_matrix;
    uint32_t* point_list;                                                          // binning: per instance
    uint8_t *bmask, *cmask;
    long long capacity;                                                            // instances the binning holds
    int recf, gx, gy, tiles;                                                       // tiles: of one view (gx * gy)
    int chunk_len, chunks;                                                         // binning: depth-sorted runs
    // Several views (V > 1): per-Gaussian regions hold V * P rows (row v * P + g = Gaussian g seen from view v), the
    // per-pixel planes and per-tile arrays hold V images stacked as one tall tile grid (view v owns tile rows
    // [v * gy, (v + 1) * gy)), and every view has its own header and depth-sort region.  view_slice() narrows the
    // buffers to one view for the per-view front end and the projection backward.
    int V, P;
    size_t sort_stride;                                                            // bytes between the views' sort regions
    uint32_t row_base;                                                             // slice: first row of the view (v * P)
    const GeomHeader* prev_header;                                                 // slice: the previous view's header or null
};

// Bit 3 of a row's clamped byte: some pixel composited the row in the forward pass (its out_weights is > 0).  The
// projection writes every row's byte with the bit clear, the forward compositor sets it.  Every other row's gradient is
// exactly zero, so the backward neither zeroes nor reads it.
constexpr unsigned kComposited = 8u;

// api.cu: view v's slice: header, sort region, per-Gaussian rows and tile ranges of that view.  The binning lists stay
// shared (the views' lists follow each other in one buffer) and the tall grid's tile order is built once for all views.
RasterBuffers view_slice(const RasterBuffers& b, int v);

// view v's {tan_fovx, tan_fovy, cx, cy}: a one-view call keeps its scalar fields (passed in), a V-view call reads row v
// of its host table
inline void view_cam(int V, const float* view_cams, int v, float& tan_fovx, float& tan_fovy, float& cx, float& cy) {
    if (V <= 1) return;
    const float* c = view_cams + 4 * v;
    tan_fovx = c[0]; tan_fovy = c[1]; cx = c[2]; cy = c[3];
}

typedef void (*stage_mark_fn)(int, cudaStream_t);
// projection.cu / projection_bwd.cu: view v of the call (its camera, per-view inputs and outputs), on view_slice(b, v)
int launch_projection(const r3dg_raster_fwd_args& a, const RasterBuffers& b, int v, cudaStream_t stream);
int launch_point_offsets(int P, const uint32_t* tiles_touched, uint32_t* out, uint32_t* state,
                         GeomHeader* ticket_header, cudaStream_t stream);
int launch_cta_order(const uint32_t* work, uint32_t* order, int n, cudaStream_t stream);
int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                        cudaStream_t stream);
// radix_sort.cu: stable sort of n (u32 key, u32 value) pairs laid out by SortLayout in `buf`
int launch_sort(void* geom_header, char* buf, const SortLayout& sl, long long n, int num_sms,
                cudaStream_t stream);
// binning.cu: depth sort + order-preserving tile binning -> point_list, bmask, zeroed cmask, ranges, num_rendered,
// tile_order, zeroed bwd_work.  launch_empty_binning: the same per-tile outputs for P == 0 (all lists empty).
int launch_binning(int P, const RasterBuffers& b, int num_sms, cudaStream_t stream, stage_mark_fn mark,
                   int* num_rendered_host, void* count_ready_event);
int launch_empty_binning(const RasterBuffers& b, cudaStream_t stream);
// the compositors' tile order over all V * tiles tiles of the tall grid (and zeroed bwd_work), after every view's binning
int launch_tile_order(const RasterBuffers& b, cudaStream_t stream);
int launch_rebuild_keys(int T, const void* ranges, const uint32_t* point_list, const float* rec, int recf,
                        long long limit, uint64_t* keys, cudaStream_t stream);
int launch_composite_forward(const r3dg_raster_fwd_args& a, const RasterBuffers& b, cudaStream_t stream,
                             stage_mark_fn mark);
// geometry = false: the appearance-only backward (r3dg_raster_backward with every geometry output NULL).  The
// compositor then leaves rows of composite_bwd_row_floats(S, false) = 4 * num_groups(S) channel gradients, and
// launch_appearance_backward turns them into dL_dcolors / dL_dfeatures / dL_dsh (or the SH factors) for all views.
int composite_bwd_row_floats(int S, bool geometry);
int launch_composite_backward(const r3dg_raster_bwd_args& a, const RasterBuffers& b, bool geometry, cudaStream_t stream);
// deterministic mode: the 2 V scale words of the compositor's rows (per view: colour / feature slots, geometry slots).
// They sit at the start of the float gradient rows' scratch region of `geom` (the call's, also for a view slice `b`),
// which the deterministic backward otherwise neither writes nor reads: its rows live in the det workspace.  That
// region holds V * P * recf >= 8 V floats.
uint32_t* raster_det_scale(const RasterBuffers& b);
// deterministic mode with absgrad (dL_dmeans2D_abs given): the 2 accumulators per row of the `rows` = V * P rows'
// absgrad sums, in det_work right behind the gradient rows' r3dg_raster_bwd_det_bytes(V * P, S)
DetAcc raster_det_abs(const r3dg_raster_bwd_args& a, size_t rows);
int launch_projection_backward(const r3dg_raster_bwd_args& a, const RasterBuffers& b, int v, cudaStream_t stream);
int launch_appearance_backward(const r3dg_raster_bwd_args& a, const RasterBuffers& b, cudaStream_t stream);

// Camera gradients: the terms of one view in the order viewmatrix [16], projmatrix [16], campos [3].  The projection
// backward writes one partial sum of them per CTA of kCamGradThreads Gaussians; launch_cam_grad_sum adds the partials
// in CTA order.
constexpr int kCamGradFloats = 35;
constexpr int kCamGradThreads = 128;
inline int cam_grad_blocks(int P) { return ((P < 1 ? 1 : P) + kCamGradThreads - 1) / kCamGradThreads; }
struct CamGradOut {
    float* out[3];                 // column k of the partials goes to the segment it falls in, [V, n[s]] per segment
    int n[3];
};
// projection_bwd.cu: out from the [V][sum n][nblk] partials in `work`, one fixed-order sum per (view, column)
int launch_cam_grad_sum(const float* work, int nblk, int V, const CamGradOut& o, cudaStream_t stream);

// surface_bwd.cu: the adjoint of the pseudo-normal / surface-xyz pass, one launch per view.  planes: [2][V][H][W] (the
// combined depth cotangents, then opacity); cam_part: [V][9][surface_grad_blocks(W, H)] or null (no camera term).
int surface_grad_blocks(int W, int H);
int launch_surface_backward(const r3dg_raster_bwd_args& a, int V, float* planes, float* cam_part, cudaStream_t stream);
// dL_dviewmatrix[v][4k + i] += the sum of view v's partials of entry 3k + i in CTA order (one launch for all views)
int launch_surface_cam_sum(const float* cam_part, int nblk, int V, float* dL_dviewmatrix, cudaStream_t stream);

size_t bvh_build_tmp_bytes(int P);
size_t bvh_packets_bytes(int P);
int launch_bvh_leaf_aabbs(int P, const float* means3D, const float* scales, const float* rotations,
                          int32_t* nodes, float* aabbs, cudaStream_t stream);
int launch_bvh_build(int P, int32_t* nodes, float* aabbs, uint64_t* morton, void* tmp, size_t tmp_bytes,
                     int num_sms, cudaStream_t stream);
int launch_bvh_trace(int P, long long num_rays, const int32_t* nodes, const float* aabbs,
                     const float* rays_o, int o_group, float o_offset, const float* rays_d,
                     const float* means3D, const float* covs3D, const float* opacities,
                     const float* normals, int32_t* num_contributes, float* rendered_opacity,
                     void* packets, size_t packets_bytes, int num_sms, cudaStream_t stream);

int launch_sample_dirs(int P, int N, const float* normals, const float* phase, float* dirs, float* areas, int num_sms, cudaStream_t stream);
int launch_bvh_bake(int P, int first_slot, int count, int N, const int32_t* nodes, const float* aabbs, const float* means3D,
                    const float* covs3D, const float* opacities, const float* normals, float o_offset,
                    int32_t* num_contributes, float* visibility, float* dirs, float* areas, void* packets,
                    size_t packets_bytes, int num_sms, cudaStream_t stream);
int launch_unpremultiply_forward(int S, long long HW, const float* feature, const float* opacity, const int32_t* n_contrib,
                                 float* out, int num_sms, cudaStream_t stream);
int launch_unpremultiply_backward(int S, long long HW, const float* feature, const float* opacity, const int32_t* n_contrib,
                                  const float* g, float* d_feature, float* d_opacity, int num_sms, cudaStream_t stream);

int launch_pack_features_forward(int P, int S, const float* means3D, const float* view, int num, const r3dg_pack_src* srcs,
                                 float* out, int num_sms, cudaStream_t stream);
int launch_pack_features_backward(int P, int S, const float* means3D, const float* view, const float* g, int num,
                                  const r3dg_pack_src* dsts, float* d_means3D, float* d_view, void* work, size_t work_bytes,
                                  int num_sms, cudaStream_t stream);

int shade_tune(const char* key, int value, int* previous);
int composite_tune(const char* key, int value, int* previous);
int composite_bwd_tune(const char* key, int value, int* previous);

// api.cu: SMs of the current device, cached per device (132, the H100 SXM count, if the query fails)
int num_sms();

// Lets kernel K launch with up to `bytes` of dynamic shared memory on the current device.  Function attributes belong
// to the device's context and a caller may drive several GPUs from one process, so the attribute is raised once per
// (kernel, device) and only when a launch needs more than an earlier one did.
constexpr int kMaxDevices = 64;
template <auto K>
inline cudaError_t allow_dyn_smem(size_t bytes) {
    static size_t allowed[kMaxDevices] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const bool cached = dev >= 0 && dev < kMaxDevices;
    if (cached && bytes <= allowed[dev]) return cudaSuccess;
    e = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess && cached) allowed[dev] = bytes;
    return e;
}

// Dynamic shared memory to request so that at most `ctas` CTAs of kernel K are resident per SM (0 when ctas <= 0 or
// the kernel's own footprint already allows no more).  The compositors are bound by their heaviest warps (a pixel
// block that composites its entries one after the other): fewer co-resident warps let those run faster while the
// total throughput stays issue-bound (tools/residency_sweep.py sweeps the setting).
template <auto K>
inline size_t residency_pad(int ctas) {
    if (ctas <= 0) return 0;
    cudaFuncAttributes fa;
    int dev = 0, smem_sm = 0, smem_blk = 0;
    if (cudaFuncGetAttributes(&fa, K) != cudaSuccess || cudaGetDevice(&dev) != cudaSuccess) return 0;
    cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    cudaDeviceGetAttribute(&smem_blk, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    const size_t fixed = fa.sharedSizeBytes + 1024;                       // static + the per-CTA system reservation
    size_t per = ((size_t)smem_sm / (size_t)ctas) & ~(size_t)127;
    if (per <= fixed) return 0;
    size_t dyn = per - fixed;
    if (fa.sharedSizeBytes + dyn > (size_t)smem_blk) dyn = (size_t)smem_blk - fa.sharedSizeBytes;
    if (allow_dyn_smem<K>(dyn) != cudaSuccess) { cudaGetLastError(); return 0; }
    return dyn;
}

// adam.cu: one launch per <= 16 parameter tensors
int launch_adam(int num, const r3dg_adam_tensor* tensors, cudaStream_t stream, int* launches);

size_t compact_tmp_bytes(int P);
int launch_compact_scan(int P, const uint8_t* keep, void* tmp, size_t tmp_bytes, int* count_host, cudaStream_t stream);
int launch_compact_rows(int P, int num, const r3dg_compact_tensor* tensors, const uint8_t* keep, const void* tmp,
                        int num_sms, cudaStream_t stream);

// densify.cu: stage-1 densification statistics and densify-and-prune; launchers validate before launching
size_t densify_tmp_bytes(int P);
int launch_densify_stats(int P, const float* vgrad, int stride, const float* ngrad, const uint8_t* filter, const float* weights,
                         const int32_t* radii, float* weights_accum, float* xyz_accum, float* normal_accum, float* denom,
                         float* max_radii2D, cudaStream_t stream);
int launch_densify_classify(int P, const float* xyz_accum, const float* normal_accum, const float* denom,
                            const float* weights_accum, const float* scaling, const float* opacity,
                            const r3dg_densify_thresholds& th, void* tmp, size_t tmp_bytes, int* totals_host,
                            cudaStream_t stream);
int launch_densify_apply(int P, const int* totals, int num, const r3dg_densify_tensor* tensors, const float* rotation,
                         const float* scaling, const float* samples, float split_recip, const void* tmp, size_t tmp_bytes,
                         int num_sms, cudaStream_t stream);

// filter3d.cu: Mip-Splatting's 3D filter sizes from the training cameras; the launcher validates before launching
size_t filter3d_tmp_bytes(int P);
int launch_filter3d(int P, int V, const float* means3D, const float* viewmatrices, const float* intrinsics, float F,
                    float* out, void* tmp, size_t tmp_bytes, int sms, cudaStream_t stream);
// mcmc.cu: MCMC densification (relocation, growth) and position noise; launchers validate before launching
size_t mcmc_tmp_bytes(int P, int n_new);
int launch_mcmc_noise(int P, float* xyz, const float* rotation, const float* scaling, const float* opacity, const float* z,
                      double scale, double k, double t, cudaStream_t stream);
int launch_mcmc_classify(int P, const float* opacity, float min_opacity, void* tmp, size_t tmp_bytes, cudaStream_t stream);
int launch_mcmc_apply(int P, int n_new, const float* u, const float* opacity, const float* scaling, double min_opacity, int n_max,
                      int num, const r3dg_densify_tensor* tensors, void* tmp, size_t tmp_bytes, int num_sms,
                      cudaStream_t stream);

size_t knn_tmp_bytes(int P);
int launch_knn(int P, const float* points, float* out, void* tmp, size_t tmp_bytes, int num_sms, cudaStream_t stream);

// ssim.cu: fused SSIM loss; both launchers validate every argument before launching anything
size_t ssim_tmp_bytes(int N, int C, int H, int W);
int launch_ssim_forward(int N, int C, int H, int W, const float* img1, const float* img2, int size_average, float* out,
                        void* tmp, size_t tmp_bytes, cudaStream_t stream);
int launch_ssim_backward(int N, int C, int H, int W, const float* img1, const float* img2, int size_average,
                         const float* dL_dout, float* dL_dimg1, cudaStream_t stream);

// smooth.cu: edge-aware smoothness and TV losses; every launcher validates its arguments before launching anything
size_t edge_aware_tmp_bytes(int Cd, int Ci, int H, int W);
int launch_edge_aware_forward(int Cd, int Ci, int H, int W, const float* data, const float* img, float* out, void* tmp,
                              size_t tmp_bytes, cudaStream_t stream);
int launch_edge_aware_backward(int Cd, int Ci, int H, int W, const float* data, const float* img, const float* dL_dout,
                               float* dL_ddata, float* dL_dimg, cudaStream_t stream);
size_t tv_tmp_bytes(int B, int H, int W);
int launch_tv_forward(int B, int H, int W, const float* x, float* out, void* tmp, size_t tmp_bytes, cudaStream_t stream);
int launch_tv_backward(int B, int H, int W, const float* x, const float* dL_dout, float* dL_dx, cudaStream_t stream);

// bilagrid.cu: bilateral-grid slice and its gradients; both launchers validate every argument before launching anything
size_t bilagrid_tmp_bytes(int G, int N, int H, int W, int GX, int GY, int L);
int launch_bilagrid_forward(int G, int N, int H, int W, int GX, int GY, int L, const float* grids, const int* ids,
                            const float* rgb, float* out, cudaStream_t stream);
int launch_bilagrid_backward(int G, int N, int H, int W, int GX, int GY, int L, const float* grids, const int* ids,
                             const float* rgb, const float* dL_dout, float* dL_drgb, float* dL_dgrids, void* tmp,
                             size_t tmp_bytes, cudaStream_t stream);

}  // namespace r3dg
