// Internal launcher declarations shared by the translation units of libr3dg_b200.so.
#pragma once
#include <cuda_runtime.h>
#include "../../include/r3dg_b200.h"
#include "common.cuh"

namespace r3dg {

typedef void (*stage_mark_fn)(int, cudaStream_t);
int launch_projection(const r3dg_raster_fwd_args& a, const GeomLayout& gl, cudaStream_t stream);
int launch_point_offsets(int P, const uint32_t* tiles_touched, uint32_t* out, uint32_t* state,
                         GeomHeader* ticket_header, cudaStream_t stream);
int launch_tile_order(const void* ranges, uint32_t* tile_order, uint32_t* bwd_work, int num_tiles, cudaStream_t stream);
int launch_cta_order(const uint32_t* work, uint32_t* order, int n, cudaStream_t stream);
int launch_mark_visible(int P, const float* means3D, const float* viewmatrix, uint8_t* present,
                        cudaStream_t stream);
// radix_sort.cu: stable sort of n (u32 key, u32 value) pairs laid out by SortLayout in `buf`
int launch_sort(void* geom_header, char* buf, const SortLayout& sl, long long n, int num_sms,
                cudaStream_t stream);
// binning.cu: depth sort + order-preserving tile binning -> point_list, ranges, num_rendered
int launch_binning(int P, int W, int H, char* geom, const GeomLayout& gl, char* img, const ImgLayout& il,
                   char* bin, const BinLayout& bl, int num_sms, cudaStream_t stream, stage_mark_fn mark,
                   int* num_rendered_host, void* count_ready_event);
int launch_rebuild_keys(int T, const void* ranges, const uint32_t* point_list, const float* rec, int recf,
                        long long limit, uint64_t* keys, cudaStream_t stream);
int launch_block_masks(int W, int H, const GeomLayout& gl, const ImgLayout& il, char* geom, char* img, char* bin,
                       const BinLayout& bl, cudaStream_t stream);
int launch_composite_forward(const r3dg_raster_fwd_args& a, const GeomLayout& gl,
                             const ImgLayout& il, char* bin, const BinLayout& bl,
                             cudaStream_t stream, stage_mark_fn mark);
int launch_composite_backward(const r3dg_raster_bwd_args& a, const GeomLayout& gl,
                              const ImgLayout& il, char* bin, const BinLayout& bl,
                              cudaStream_t stream);
int launch_projection_backward(const r3dg_raster_bwd_args& a, const GeomLayout& gl,
                               cudaStream_t stream);

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
                                  const r3dg_pack_src* dsts, float* d_means3D, int num_sms, cudaStream_t stream);

int shade_tune(const char* key, int value, int* previous);
int composite_tune(const char* key, int value, int* previous);
int composite_bwd_tune(const char* key, int value, int* previous);

// Dynamic shared memory to request so that at most `ctas` CTAs of `kernel` are resident per SM (0 when ctas <= 0 or
// the kernel's own footprint already allows no more).  The compositors are bound by their heaviest warps (a pixel
// block that composites its entries one after the other): fewer co-resident warps let those run faster while the
// total throughput stays issue-bound (tools/residency_sweep.py sweeps the setting).
template <typename K>
inline size_t residency_pad(K kernel, int ctas) {
    if (ctas <= 0) return 0;
    cudaFuncAttributes fa;
    int dev = 0, smem_sm = 0, smem_blk = 0;
    if (cudaFuncGetAttributes(&fa, kernel) != cudaSuccess || cudaGetDevice(&dev) != cudaSuccess) return 0;
    cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
    cudaDeviceGetAttribute(&smem_blk, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    const size_t fixed = fa.sharedSizeBytes + 1024;                       // static + the per-CTA system reservation
    size_t per = ((size_t)smem_sm / (size_t)ctas) & ~(size_t)127;
    if (per <= fixed) return 0;
    size_t dyn = per - fixed;
    if (fa.sharedSizeBytes + dyn > (size_t)smem_blk) dyn = (size_t)smem_blk - fa.sharedSizeBytes;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn) != cudaSuccess) { cudaGetLastError(); return 0; }
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

}  // namespace r3dg
