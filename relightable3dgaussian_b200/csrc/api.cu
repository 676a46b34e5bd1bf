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

namespace {
int g_num_sms[64] = {0};            // per device (the caller may drive several GPUs from one process)
int num_sms() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;   // H100 SXM
    if (g_num_sms[dev] == 0) {
        int n = 0;
        g_num_sms[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
    }
    return g_num_sms[dev];
}
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
}  // namespace

extern "C" {

const char* r3dg_version(void) { return "r3dg_b200 0.1 sm_90a"; }

size_t r3dg_raster_geom_bytes(int P, int S) { return GeomLayout(P < 1 ? 1 : P, S).total; }
size_t r3dg_raster_img_bytes(int W, int H) { return ImgLayout(W, H).total; }
size_t r3dg_raster_binning_bytes(long long capacity) { return bin_bytes_for_capacity(capacity < 1 ? 1 : capacity); }
size_t r3dg_raster_img_n_contrib_offset(int W, int H) { return ImgLayout(W, H).n_contrib; }
size_t r3dg_raster_fwd_det_bytes(int P) { return align_up((size_t)(P < 1 ? 1 : P) * 8, 256); }
size_t r3dg_raster_bwd_det_bytes(int P, int S) { return det_bytes((size_t)(P < 1 ? 1 : P) * rec_floats(S < 0 ? 0 : S)); }

int r3dg_det_sum_host(long long n, const float* terms, float* out) {
    if (n < 0 || (n > 0 && !terms) || !out) return R3DG_ERR_BAD_ARG;
    uint64_t lo = 0, mid = 0, hi = 0;
    uint32_t flag = 0;
    for (long long i = 0; i < n; ++i) {
        const DetTerm t = det_term(terms[i]);
        lo += t.lo; mid += t.mid; hi += t.hi; flag |= t.flag;
    }
    *out = det_value(lo, mid, hi, flag);
    return 0;
}

int r3dg_raster_forward(const r3dg_raster_fwd_args* a, r3dg_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!a || a->P < 0 || a->W <= 0 || a->H <= 0 || a->S < 0) return R3DG_ERR_BAD_ARG;
    if (a->S > R3DG_MAX_S_FWD) return R3DG_ERR_UNSUPPORTED;
    if (a->P > 0 && ((a->shs == nullptr) == (a->colors_precomp == nullptr))) return R3DG_ERR_BAD_ARG;
    if (a->P > 0 && (a->cov3D_precomp == nullptr) && (a->scales == nullptr || a->rotations == nullptr)) return R3DG_ERR_BAD_ARG;
    if (a->shs && a->M > 16) return R3DG_ERR_UNSUPPORTED;
    const GeomLayout gl(a->P < 1 ? 1 : a->P, a->S);
    const ImgLayout il(a->W, a->H);
    if (a->geom_bytes < gl.total || a->img_bytes < il.total) return R3DG_ERR_BAD_ARG;
    if (a->deterministic && (!a->det_work || a->det_work_bytes < r3dg_raster_fwd_det_bytes(a->P))) return R3DG_ERR_BAD_ARG;
    const long long capacity = bin_capacity_for_bytes(a->binning_bytes);
    if (capacity < 1) return R3DG_ERR_BAD_ARG;
    const BinLayout bl(capacity);
    char* geom = (char*)a->geom;
    char* img = (char*)a->img;
    char* bin = (char*)a->binning;
    R3DG_CUDA_TRY(cudaMemsetAsync(geom + gl.header, 0, sizeof(GeomHeader), stream));
    int rc = 0;
    auto mark = [](int i, cudaStream_t s) { prof_mark(true, i, s); };
    prof_mark(true, 0, stream);
    if (a->P > 0) {
        if ((rc = launch_projection(*a, gl, stream)) != 0) return rc;
        prof_mark(true, 1, stream);
        if ((rc = launch_binning(a->P, a->W, a->H, geom, gl, img, il, bin, bl, num_sms(), stream, mark, a->num_rendered_host,
                                 a->count_ready_event)) != 0) return rc;
        g_launches += 1 + (1 + R3DG_SORT_MAX_PASSES) + 4;   // project; histogram + radix passes; count, colsum + starts, apply, scatter
    } else {
        if ((rc = launch_empty_binning(a->W, a->H, geom, gl, img, il, stream)) != 0) return rc;
        for (int i = 1; i <= 4; ++i) prof_mark(true, i, stream);
        g_launches += 1;                                    // starts (empty ranges, tile order)
    }
    prof_mark(true, 5, stream);
    if ((rc = launch_composite_forward(*a, gl, il, bin, bl, stream, mark)) != 0) return rc;
    prof_mark(true, 7, stream);
    g_launches += 1 + (a->computer_pseudo_normal ? 1 : 0) + (a->deterministic && a->P > 0 ? 1 : 0);   // composite, normals, weights
    if (g_prof.on) g_prof.fwd_calls++;
    if (a->P == 0) {      // (P > 0: the count was written, and the event recorded, as soon as the binning offsets existed)
        if (a->num_rendered_host) R3DG_CUDA_TRY(cudaMemcpyAsync(a->num_rendered_host, geom + gl.header, sizeof(int), cudaMemcpyDeviceToHost, stream));
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
    if (a->deterministic && (!a->det_work || a->det_work_bytes < r3dg_raster_bwd_det_bytes(a->P, a->S))) return R3DG_ERR_BAD_ARG;
    if (a->P == 0) return 0;
    const GeomLayout gl(a->P, a->S);
    const ImgLayout il(a->W, a->H);
    if (a->geom_bytes < gl.total || a->img_bytes < il.total) return R3DG_ERR_BAD_ARG;
    const long long capacity = bin_capacity_for_bytes(a->binning_bytes);
    if (capacity < 1) return R3DG_ERR_BAD_ARG;
    const BinLayout bl(capacity);
    char* bin = (char*)a->binning;
    int rc = 0;
    prof_mark(false, 8, stream);
    if ((rc = launch_composite_backward(*a, gl, il, bin, bl, stream)) != 0) return rc;
    prof_mark(false, 9, stream);
    if ((rc = launch_projection_backward(*a, gl, stream)) != 0) return rc;
    prof_mark(false, 10, stream);
    g_launches += 3;   // CTA order, composite, projection
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
                                const r3dg_pack_src* dsts, float* dL_dmeans3D, r3dg_stream_t stream) {
    if (num > 0 && !dsts) return R3DG_ERR_BAD_ARG;
    g_launches += P > 0 ? 1 : 0;
    return launch_pack_features_backward(P, S, means3D, viewmatrix, dL_dout, num, dsts, dL_dmeans3D, num_sms(), (cudaStream_t)stream);
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
    const int rc = launch_densify_apply(P, totals, num_tensors, tensors, rotation, scaling, samples, split_recip, tmp, tmp_bytes,
                                        num_sms(), (cudaStream_t)stream);
    if (rc == 0 && P > 0 && num_tensors > 0) g_launches += 1;
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
}  // namespace

long long r3dg_raster_debug_copy(int id, int P, int S, int W, int H, const void* geom_, const void* img_,
                                 const void* bin_, size_t binning_bytes, void* dst, long long max_bytes,
                                 r3dg_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    const GeomLayout gl(P < 1 ? 1 : P, S);
    const ImgLayout il(W, H);
    const char* geom = (const char*)geom_;
    const char* img = (const char*)img_;
    const char* bin = (const char*)bin_;
    const size_t HW = (size_t)W * H;
    const int tiles = ((W + R3DG_TILE - 1) / R3DG_TILE) * ((H + R3DG_TILE - 1) / R3DG_TILE);
    const float* rec = (const float*)(geom + gl.rec);
    const uint32_t* tt = (const uint32_t*)(geom + gl.tiles_touched);
    const int nb = (P + 255) / 256;
    auto copy = [&](const void* src, size_t n) -> long long {
        if ((long long)n > max_bytes) n = (size_t)max_bytes;
        if (cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, stream) != cudaSuccess) return -2;
        return (long long)n;
    };
    switch (id) {
        case 0: if (max_bytes < 4LL * P) return -1; if (P) unpack_rec_kernel<<<nb, 256, 0, stream>>>(P, gl.recf, 0, rec, tt, (float*)dst); return 4LL * P;
        case 1: if (max_bytes < 3LL * P) return -1; if (P) unpack_clamped_kernel<<<nb, 256, 0, stream>>>(P, (const uint8_t*)(geom + gl.clamped), tt, (uint8_t*)dst); return 3LL * P;
        case 3: if (max_bytes < 8LL * P) return -1; if (P) unpack_rec_kernel<<<nb, 256, 0, stream>>>(P, gl.recf, 3, rec, tt, (float*)dst); return 8LL * P;
        case 5: if (max_bytes < 16LL * P) return -1; if (P) unpack_rec_kernel<<<nb, 256, 0, stream>>>(P, gl.recf, 5, rec, tt, (float*)dst); return 16LL * P;
        case 6: if (max_bytes < 12LL * P) return -1; if (P) unpack_rec_kernel<<<nb, 256, 0, stream>>>(P, gl.recf, 6, rec, tt, (float*)dst); return 12LL * P;
        case 7: return copy(geom + gl.tiles_touched, 4 * (size_t)P);
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
        case 13: return copy(img + il.final_T, 4 * HW);
        case 14: return copy(img + il.n_contrib, 4 * HW);
        case 15: return copy(img + il.ranges, 8 * (size_t)tiles);
        case 16: return copy(img + il.bwd_work, 8 * (size_t)tiles);
        case 17: return copy(img + il.bwd_order, 8 * (size_t)tiles);
        case 20: return copy(geom + gl.brects, 8 * (size_t)P);
        case 9: case 10: case 18: case 19: {
            const long long capacity = bin_capacity_for_bytes(binning_bytes);
            if (capacity < 1) return -1;
            const BinLayout bl(capacity);
            // caller limits the copy to R entries through max_bytes
            if (id == 9) return copy(bin + bl.point_list, std::min((size_t)max_bytes, (size_t)capacity * 4));
            if (id == 18) return copy(bin + bl.bmask, std::min((size_t)max_bytes, (size_t)capacity));
            if (id == 19) return copy(bin + bl.cmask, std::min((size_t)max_bytes, (size_t)capacity));
            // reference binningState.point_list_keys (sorted): rebuilt from the lists
            const long long limit = std::min(max_bytes / 8, capacity);
            if (launch_rebuild_keys(tiles, img + il.ranges, (const uint32_t*)(bin + bl.point_list), rec, gl.recf, limit,
                                    (uint64_t*)dst, stream) != 0) return -2;
            return limit * 8;
        }
    }
    return -1;
}

}  // extern "C"
