/*
 * r3dg_b200 — C ABI of the H100-native (sm_90a) relightable-Gaussian rasterizer hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b): plain pointers and sizes, no torch types, an
 * explicit CUDA stream, caller-allocated memory, no hidden allocation, errors returned as
 * negative cudaError_t (never thrown).  Every entry point names the reference interface it
 * replaces; the Python host side (relightable3dgaussian_b200/_C_raster.py) rebuilds the exact
 * tuples of the reference's pybind module `r3dg_rasterization._C` on top of it.
 *
 * All pointers are DEVICE pointers unless stated otherwise; optional inputs are NULL when absent
 * (the reference signals absence with an empty tensor whose data_ptr is null,
 * r3dg-rasterization/cuda_rasterizer/forward.cu:206,242).
 */
#ifndef R3DG_B200_H_
#define R3DG_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* r3dg_stream_t; /* == cudaStream_t */

#define R3DG_OK 0
#define R3DG_ERR_BAD_ARG (-10001)
#define R3DG_ERR_UNSUPPORTED (-10002)

/* ------------------------------------------------------------------------------------------
 * Work-buffer sizing.  Replaces CudaRasterizer::required<GeometryState/ImageState/BinningState>
 * (r3dg-rasterization/cuda_rasterizer/rasterizer_impl.h:67-73, rasterizer_impl.cu:155-195).
 * The three buffers are opaque blobs that round-trip from forward to backward exactly like the
 * reference's geomBuffer / imgBuffer / binningBuffer (rasterize_points.cu:83-90,136-140).
 * `capacity` is the number of (tile, Gaussian) instances the binning buffer can hold.
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_raster_geom_bytes(int P, int S);
size_t r3dg_raster_img_bytes(int W, int H);
size_t r3dg_raster_binning_bytes(long long capacity);
/* Byte offset of the int32 n_contrib[H,W] plane inside the image buffer: the reference returns
 * n_contrib as a view of imgBuffer (rasterize_points.cu:136-139) and so does the host glue. */
size_t r3dg_raster_img_n_contrib_offset(int W, int H);
/* The same for a call that renders V views (the `V` field below); V = 1 gives the sizes above.  The deterministic
 * workspaces of such a call are r3dg_raster_fwd_det_bytes(V * P) and r3dg_raster_bwd_det_bytes(V * P, S). */
size_t r3dg_raster_views_geom_bytes(int P, int S, int V);
size_t r3dg_raster_views_img_bytes(int W, int H, int V);
size_t r3dg_raster_views_img_n_contrib_offset(int W, int H, int V);
#define R3DG_MAX_VIEWS 64

typedef struct r3dg_raster_fwd_args {
    int P, S, D, M, W, H;          /* Gaussians, feature channels, SH degree, SH coeffs, image */
    const float* background;       /* [3] */
    const float* means3D;          /* [P,3] */
    const float* shs;              /* [P,M,3] or NULL */
    const float* colors_precomp;   /* [P,3]  or NULL (exactly one of shs / colors_precomp) */
    const float* features;         /* [P,S]  or NULL when S == 0 */
    const float* opacities;        /* [P] */
    const float* scales;           /* [P,3]  or NULL */
    const float* rotations;        /* [P,4]  or NULL; 16-byte aligned (read as float4), else R3DG_ERR_BAD_ARG */
    const float* cov3D_precomp;    /* [P,6]  or NULL (exactly one of scales+rotations / cov3D) */
    const float* viewmatrix;       /* [16] world->view, stored transposed (scene/cameras.py:62) */
    const float* projmatrix;       /* [16] full projection, stored transposed */
    const float* campos;           /* [3] */
    float scale_modifier, tan_fovx, tan_fovy, cx, cy;
    int prefiltered, computer_pseudo_normal, debug;
    /* outputs (need not be initialised; every element is written) */
    float* out_color;              /* [3,H,W] */
    float* out_opacity;            /* [1,H,W] */
    float* out_depth;              /* [1,H,W] */
    float* out_feature;            /* [S,H,W] */
    float* out_normal;             /* [3,H,W] */
    float* out_surface_xyz;        /* [3,H,W] */
    float* out_weights;            /* [P] */
    int* radii;                    /* [P] */
    int* n_contrib;                /* [H,W] */
    /* opaque work buffers */
    void* geom;   size_t geom_bytes;
    void* img;    size_t img_bytes;
    void* binning; size_t binning_bytes;
    /* Pinned HOST int receiving num_rendered (may be NULL): page-locked memory is written directly by the
     * binning kernel that computes the count, other host memory by an async copy on `stream`.
     * num_rendered > capacity means the binning buffer was too small: outputs are invalid and
     * the call must be repeated with a larger buffer (nothing out of bounds is ever written). */
    int* num_rendered_host;
    /* optional cudaEvent_t: recorded on `stream` right after the write into num_rendered_host has been enqueued, which
     * happens as soon as the instance count exists on the device (after the binning offsets, ~1/4 into the forward) —
     * a host that waits on this event instead of the stream gets the count while the compositor is still running and
     * can already enqueue what follows the forward.  NULL: not used. */
    void* count_ready_event;
    /* Several views of the same Gaussians in one call.  V = 0 or 1: the single view described above.  With
     * 1 < V <= R3DG_MAX_VIEWS: background [V,3], viewmatrix [V,16], projmatrix [V,16] and campos [V,3] hold one row per
     * view; view_cams is a HOST array [V][4] of {tan_fovx, tan_fovy, cx, cy} (the scalar fields are not used); every
     * image output gains a leading V (out_color [V,3,H,W], ..., n_contrib [V,H,W]), out_weights and radii are [V,P];
     * num_rendered_host receives V ints, the instance count of each view (their sum > capacity = overflow).
     * features_per_view / colors_per_view: features is [V,P,S] / colors_precomp is [V,P,3] (0: shared [P,...]).
     * Every view's images are those of a one-view call with its camera.  V * P must stay below 2^30. */
    int V;
    const float* view_cams;
    int features_per_view, colors_per_view;
    /* 3D smoothing filter (Mip-Splatting's 3D filter; optional, NULL = off, the default): [P] filter sizes f >= 0, one
     * per Gaussian and shared by every view of the call (r3dg_filter3d_compute).  Each Gaussian is drawn with scales
     * s'_k = sqrt(s_k^2 + f^2) and opacity o' = o * coef, coef = sqrt((r_0 r_1) r_2), r_k = s_k^2 / s'_k^2 (1 when
     * s'_k = 0): the covariance dilated by f^2 I keeps the Gaussian's integrated weight.  Every operation is a
     * correctly rounded fp32 operation in that order (q_k = s_k s_k, g = f f, e_k = q_k + g, s'_k = sqrt(e_k),
     * r_k = q_k / e_k), so a call with the filter equals, bit for bit, a call without it on (s', o') computed the same
     * way.  scale_modifier multiplies s'.  With `antialiasing`, the record holds o' rho.  f = 0 gives s' = |s| and
     * coef = 1 (for s = 0 and every s whose square is a normal float).  With cov3D_precomp: R3DG_ERR_BAD_ARG before
     * any launch. */
    const float* filter_3d;
    /* Antialiased mode (the opacity-compensated screen-space filter of upstream 3DGS and gsplat).  Non-zero: with
     * a0, b, c0 the 2D covariance before the fixed 0.3 px^2 dilation and a1 = a0 + 0.3, c1 = c0 + 0.3, every Gaussian's
     * opacity is multiplied by rho = sqrt(max(r, 2.5e-5)), r = (a0 c0 - b^2) / (a1 c1 - b^2) (r = 0 when a0 c0 - b^2
     * <= 0), so that the dilated Gaussian keeps the integrated weight of the undilated one.  The compensated opacity
     * replaces the opacity in the record every compositor reads (and so in out_weights and the block pre-filter);
     * the conic, radius, tile rectangle, depth key and colours are those of 0.  0 = the default path. */
    int antialiasing;
    /* Deterministic mode (torch.use_deterministic_algorithms(True)): non-zero = sums that float atomics would make
     * depend on warp arrival order are accumulated in fixed point in `det_work` (see DETERMINISTIC MODE below);
     * det_work: device workspace of at least r3dg_raster_fwd_det_bytes(P) bytes, zeroed by the call.  0 = the default path (det_work unused). */
    int deterministic;
    void* det_work; size_t det_work_bytes;
} r3dg_raster_fwd_args;

/* Replaces CudaRasterizer::Rasterizer::forward (rasterizer.h:34-65, rasterizer_impl.cu:199-380)
 * == `_C.rasterize_gaussians` (rasterize_points.cu:36-141).  Enqueues the whole forward on
 * `stream` without any host synchronisation. */
int r3dg_raster_forward(const r3dg_raster_fwd_args* args, r3dg_stream_t stream);

typedef struct r3dg_raster_bwd_args {
    int P, S, D, M, W, H;
    const float* background;
    const float* means3D;
    const float* shs;
    const float* colors_precomp;
    const float* features;
    const float* scales;
    const float* rotations;        /* 16-byte aligned, as in the forward */
    const float* cov3D_precomp;
    const float* viewmatrix;
    const float* projmatrix;
    const float* campos;
    float scale_modifier, tan_fovx, tan_fovy;
    int backward_geometry, debug;
    /* cotangents, contiguous */
    const float* dL_dout_color;    /* [3,H,W] */
    const float* dL_dout_opacity;  /* [1,H,W] */
    const float* dL_dout_depth;    /* [1,H,W] */
    const float* dL_dout_feature;  /* [S,H,W] */
    /* gradients out (need not be initialised; every element is written) */
    float* dL_dmeans2D;            /* [P,3]  (depth gradient in .z) */
    float* dL_dcolors;             /* [P,3] */
    float* dL_dopacity;            /* [P] */
    float* dL_dmeans3D;            /* [P,3] */
    float* dL_dfeatures;           /* [P,S] */
    float* dL_dcov3D;              /* [P,6] */
    float* dL_dsh;                 /* [P,M,3]; may be NULL when dL_dsh_factor is given */
    float* dL_dscales;             /* [P,3] */
    float* dL_drotations;          /* [P,4]; 16-byte aligned (written as float4), else R3DG_ERR_BAD_ARG */
    float* dL_dsh_factor;          /* [P,3] or NULL: the view's rank-1 factor of dL_dsh, see r3dg_sh_grad_from_factors */
    /* APPEARANCE-ONLY MODE (for training with frozen geometry): every geometry output NULL — dL_dmeans2D,
     * dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dscales, dL_drotations and the three camera gradients.  The backward
     * then computes only the colour / feature / SH gradients: the compositor forms and reduces only the 3 + S colour
     * and feature components of each entry (no dL/dalpha), and no covariance, mean or camera chain runs.
     *   - Some of the six per-Gaussian geometry outputs NULL and others not, or a camera gradient with all six NULL,
     *     returns R3DG_ERR_BAD_ARG before any launch.
     *   - dL_dcolors, dL_dfeatures and dL_dsh may each be NULL (not computed); all three NULL returns
     *     R3DG_ERR_BAD_ARG.  Every element of a requested output is written, rows no pixel composited as +0.  (P = 0
     *     writes no per-Gaussian output and refuses none of these combinations.)
     *   - The cotangents of opacity, depth, pseudo-normal and surface-xyz are ignored (they may be NULL): those outputs
     *     depend only on the geometry and have no appearance gradient.
     *   - One view and V views (per-view features / colors included) and the deterministic mode work as in the full
     *     backward, with the same workspace; a requested gradient equals the full backward's (bitwise in deterministic
     *     mode).  With `shs`, dL_dsh_factor, when given, receives each view's factor exactly as in the full backward;
     *     V > 1 with dL_dsh requires it, as there.
     * The per-view projection backward is replaced by one launch over all views. */
    /* work buffers written by the matching forward */
    void* geom;   size_t geom_bytes;
    void* img;    size_t img_bytes;
    void* binning; size_t binning_bytes;
    /* Several views (see r3dg_raster_fwd_args; the same V, camera rows, view_cams and per-view flags as the forward).
     * The cotangents are [V,...]; dL_dmeans2D is [V,P,3]; dL_dfeatures / dL_dcolors are [V,P,*] when the input was per
     * view.  Every other gradient is the sum over the views, accumulated in fp32 in view order (g_0 + g_1 + ...).
     * With `shs`, dL_dsh_factor [V,P,3] is required: each view writes its rank-1 factor there and dL_dsh is rebuilt
     * from the factors (r3dg_sh_grad_from_factors, scale 1). */
    int V;
    const float* view_cams;
    int features_per_view, colors_per_view;
    /* Camera gradients (optional; all three NULL = none, the default).  One row per view, never summed over views:
     *   dL_dviewmatrix [V,16] and dL_dprojmatrix [V,16] in the element order of `viewmatrix` / `projmatrix`, i.e. the
     *   memory of torch's world_view_transform / full_proj_transform: element 4j + k is matrix[j][k];
     *   dL_dcampos [V,3].
     * Entries the projection never reads (column 3 of viewmatrix, column 2 of projmatrix) are exactly 0, and so is the
     * whole row of a view in which every Gaussian is culled, or of every view when P = 0.  The gradients are those of
     * the projection's closed form: through t = [m,1] viewmatrix and T = W J into the 2D covariance and depth, through
     * the homogeneous projection into the 2D mean (with the forward's + 1e-7), and through the SH view direction.  Each
     * CTA of the projection backward sums its Gaussians' terms in a fixed order into cam_work, and one more launch adds
     * those partial sums in CTA order: no float atomics, so equal gradient rows give equal bits (in deterministic mode
     * the camera gradients are bitwise reproducible).
     * cam_work: device workspace of at least r3dg_raster_cam_grad_bytes(P, V) bytes.  Only some of the three outputs,
     * or too small a workspace, returns R3DG_ERR_BAD_ARG before anything is launched. */
    float* dL_dviewmatrix;
    float* dL_dprojmatrix;
    float* dL_dcampos;
    void* cam_work; size_t cam_work_bytes;
    /* Gradients of the pseudo-normal and surface-xyz outputs (optional; both cotangents NULL = none, the default: the
     * forward's out_normal / out_surface_xyz are then constants, as in the reference).
     *   dL_dout_normal, dL_dout_surface_xyz: [V,3,H,W]; either may be NULL, which means zero.
     *   fwd_opacity, fwd_depth: [V,1,H,W], the forward's out_opacity / out_depth (required with either cotangent).
     *   cx, cy: the principal point of a call with V = 0 or 1, which must be set (a call with V > 1 reads each view's
     *           from view_cams; there these fields are unused).
     * One launch per view runs the adjoint of the forward's surface/normal pass: it adds the cotangents' pull-back to
     * dL_dout_depth and dL_dout_opacity, writes the sums to surface_work, and the backward compositor runs unchanged on
     * them.  With dL_dviewmatrix, the pseudo-normal's term sum_pixels g_normal_k N_i is added to element 4k + i after
     * the projection's term, summed in a fixed order (one more launch).  No float atomics: bitwise reproducible.
     * surface_work: device workspace of at least r3dg_raster_surface_grad_bytes(W, H, V) bytes, laid out as
     *   [0]                                   float [2][V][H][W]: the combined depth cotangents of all views, then the
     *                                         combined opacity cotangents (the planes the compositor consumed);
     *   [align256(8 V H W)]                   float [V][9][blocks]: per-CTA partials of the camera term, blocks =
     *                                         ceil(W / 32) ceil(H / 8).
     * A cotangent without both forward images, or a missing or too small workspace, returns R3DG_ERR_BAD_ARG before
     * anything is launched.  P = 0 launches nothing (every gradient is zero). */
    const float* dL_dout_normal;
    const float* dL_dout_surface_xyz;
    const float* fwd_opacity;
    const float* fwd_depth;
    float cx, cy;
    void* surface_work; size_t surface_work_bytes;
    /* 3D smoothing filter (see r3dg_raster_fwd_args): NULL, or [P] holding the matching forward's values, like
     * scale_modifier.  `opacities` [P] is the forward's opacity o, required with filter_3d (the record holds o coef,
     * and coef may be 0 or subnormal, so o is not recovered from it).  Live rows then get dL_dopacity = coef dL/do' and
     * dL_dscales_k = dL/ds'_k s_k / s'_k + o dL/do' dcoef/ds_k (s_k / s'_k = 1 where s'_k = 0); there is no gradient
     * with respect to f.  filter_3d with cov3D_precomp, or without opacities, returns R3DG_ERR_BAD_ARG before any
     * launch.  The appearance-only mode ignores both fields. */
    const float* filter_3d;
    const float* opacities;
    /* Absolute screen-space gradients (absgrad, AbsGS / gsplat's absgrad=True; optional, NULL = none, the default):
     * [P,2] ([V,P,2] for V views), next to dL_dmeans2D and in its units (0.5 W and 0.5 H per pixel): per Gaussian and
     * view, sum over pixels of |dL/dmean2D.x| and of |dL/dmean2D.y|, each pixel's term taken before the pixel sum, so
     * that pixels pulling a Gaussian in opposite directions do not cancel.  +0 for rows no pixel composited; every
     * element is written.  It includes the pseudo-normal / surface-xyz pull-back and the antialiased mode's
     * compensated opacity as dL_dmeans2D does.  The appearance-only mode ignores it.  In deterministic mode det_work
     * must then hold r3dg_raster_bwd_det_bytes(V * P, S) + r3dg_raster_bwd_det_absgrad_bytes(V * P) bytes (too small
     * returns R3DG_ERR_BAD_ARG before any launch); the sums are fixed-point sums of the geometry class. */
    float* dL_dmeans2D_abs;
    /* Antialiased mode: must equal the matching forward's (zero or non-zero), like scale_modifier and the matrices;
     * the backward reads the compensated opacity from the forward's record and differentiates rho too.  dL_dopacity is
     * then rho times the gradient of the compensated opacity, and rho's dependence on the 2D covariance reaches
     * dL_dcov3D, dL_dscales, dL_drotations, dL_dmeans3D and dL_dviewmatrix.  The appearance-only mode ignores it. */
    int antialiasing;
    /* Deterministic mode (torch.use_deterministic_algorithms(True)): non-zero = sums that float atomics would make
     * depend on warp arrival order are accumulated in fixed point in `det_work` (see DETERMINISTIC MODE below);
     * det_work: device workspace of at least r3dg_raster_bwd_det_bytes(P, S) bytes, zeroed by the call.  0 = the default path (det_work unused). */
    int deterministic;
    void* det_work; size_t det_work_bytes;
} r3dg_raster_bwd_args;

/* Replaces CudaRasterizer::Rasterizer::backward (rasterizer.h:67-100, rasterizer_impl.cu:384-491)
 * == `_C.rasterize_gaussians_backward` (rasterize_points.cu:143-235). */
int r3dg_raster_backward(const r3dg_raster_bwd_args* args, r3dg_stream_t stream);
/* Workspace of the camera gradients of a V-view backward (r3dg_raster_bwd_args.cam_work); P = 0 and V < 1 are sized
 * as 1.  r3dg_raster_cam_grad_bytes(P, 1) also covers the workspace of r3dg_pack_features_backward. */
size_t r3dg_raster_cam_grad_bytes(int P, int V);
/* Workspace of the pseudo-normal / surface-xyz gradients of a V-view backward (r3dg_raster_bwd_args.surface_work):
 * align256(8 V W H) + align256(36 V ceil(W / 32) ceil(H / 8)) bytes; W, H and V below 1 are sized as 1. */
size_t r3dg_raster_surface_grad_bytes(int W, int H, int V);

/* Multi-GPU exchange step (SURVEY.md §8e; the reference is single-GPU).  For one view the SH
 * gradient is rank-1 per Gaussian: dL_dsh[g,k,:] = basis_k(normalize(mean_g - campos)) * f[g,:]
 * with f = dL_dRGB gated by the forward's clamp flags (backward.cu:20-139) and zero for culled
 * Gaussians — r3dg_raster_backward writes f to `dL_dsh_factor`.  Instead of all-reducing the dense
 * [P,M,3] tensor (192 B per Gaussian) the ranks all-gather f (12 B per Gaussian and view) and every
 * rank rebuilds the reduced gradient locally:
 *     dL_dsh[g,k,c] = scale * sum_v basis_k(normalize(means3D[g] - campos[v])) * factors[v][g][c]
 * for k < (D+1)^2 (zero above), v = 0..num_views-1 in order (deterministic, identical on every
 * rank).  campos: [num_views,3]; factors: [num_views,P,3]; dL_dsh: [P,M,3] (every element written). */
int r3dg_sh_grad_from_factors(int P, int D, int M, int num_views, const float* means3D,
                              const float* campos, const float* factors, float scale,
                              float* dL_dsh, r3dg_stream_t stream);

/* The same exchange as ONE kernel over NVLink peer memory (no NCCL call): the per-view factors and the dense
 * per-Gaussian gradient section live in symmetric buffers mapped into every rank (the caller allocates and
 * rendezvouses them, e.g. torch.distributed._symmetric_memory).  The launch
 *   (a) rebuilds dL_dsh as r3dg_sh_grad_from_factors does, loading view v's 12 B per Gaussian straight from rank v's
 *       buffer (coalesced P2P loads: the transfer overlaps the outer-product math), scale = 1/world;
 *   (b) replaces the section dense[rank][0..n_dense) on EVERY rank by its mean over the ranks: rank r reduces slice r
 *       with `multimem.ld_reduce` through the NVSwitch multicast mapping `dense_multicast` (in-switch reduction) and
 *       writes it back to all ranks with `multimem.st`; with dense_multicast == NULL it falls back to peer loads/stores.
 * The caller must order it between two cross-rank barriers (all ranks' backward kernels done before; all ranks'
 * exchange kernels done before anyone reads the dense section or overwrites a factor buffer).  n_dense: floats,
 * a multiple of 4, 16-byte aligned sections.  world <= 64. */
typedef struct r3dg_exchange_args {
    int P, D, M, world, rank;
    const float* means3D;          /* [P,3] (replicated) */
    const float* campos;           /* [world,3] camera centres of the ranks' views */
    const float* factors[64];      /* [v]: rank v's [P,3] factor buffer (peer pointer; [rank] is local) */
    float* dL_dsh;                 /* [P,M,3] local output */
    long long n_dense;             /* 0: no dense job */
    float* dense[64];              /* [v]: rank v's dense section (peer pointer) */
    float* dense_multicast;        /* multicast address of the section or NULL */
} r3dg_exchange_args;
int r3dg_exchange_p2p(const r3dg_exchange_args* args, r3dg_stream_t stream);

/* Replaces Rasterizer::markVisible (rasterizer_impl.cu:141-153) == `_C.mark_visible`
 * (rasterize_points.cu:237-256).  present: uint8/bool [P]. */
int r3dg_mark_visible(int P, const float* means3D, const float* viewmatrix,
                      const float* projmatrix, uint8_t* present, r3dg_stream_t stream);

/* Debug / parity introspection of the opaque buffers after a forward (SURVEY.md §8c asks for the
 * same visibility the reference's obtain() layout gives).  Copies one named intermediate into
 * `dst` (device pointer) as a dense array in the REFERENCE's element layout.
 * ids: 0 depths f32[P] | 1 clamped u8[3P] | 3 means2D f32[2P] | 5 conic_opacity f32[4P]
 *      6 rgb f32[3P] | 7 tiles_touched u32[P] | 8 point_offsets u32[P] | 9 point_list u32[R]
 *      10 point_list_keys u64[R] | 13 final_T f32[HW] | 14 n_contrib i32[HW] | 15 ranges u32[2T]
 *      (ours only) 16 bwd_work u32[2T]: entries composited by the busiest warp of each half-tile
 *      CTA | 17 bwd_order u32[2T]: the backward compositor's launch order (valid after a backward)
 *      | 18 bmask u8[R]: per list entry, bit b = 8x4 pixel block b of the entry's tile (row b >> 1,
 *      column b & 1) meets the Gaussian's block rectangle | 19 cmask u8[R]: per list entry, bit b =
 *      block b composited the entry in the forward | 20 brects u32[2P]: per Gaussian the inclusive
 *      block rectangle {bx0 | bx1 << 16, by0 | by1 << 16} (empty when bx0 > bx1) | 22 composited
 *      u8[P]: 1 when some pixel composited the Gaussian (the backward reads and zeroes its rows only)
 *      (9, 18, 19: the copy stops at max_bytes, pass R entries' worth)
 * Returns bytes written or a negative error. */
long long r3dg_raster_debug_copy(int id, int P, int S, int W, int H, const void* geom,
                                 const void* img, const void* binning, size_t binning_bytes,
                                 void* dst, long long max_bytes, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * BVH visibility: LBVH over the Gaussians' 3-sigma boxes + opacity ray trace.
 * Replaces the reference's `bvh_tracing._C` (bvh/src/bindings.cpp:8-13, bvh/include/bvh.h).
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_bvh_build_tmp_bytes(int P);
size_t r3dg_bvh_trace_tmp_bytes(int P);

/* Fused replacement of the PyTorch prologue of RayTracer.__init__ (bvh/__init__.py:29-57):
 * fills nodes i32[2P-1,5] (all -1, count column 0 for internal / 1 for leaf nodes) and aabbs
 * f32[2P-1,6] (internal: +1e5/-1e5, leaf i at row P-1+i: box of the 8 corners mu +- 3 s_a a +- ...),
 * with the same op-by-op fp32 rounding as the PyTorch expression.  rotations [P,4] must be 16-byte
 * aligned (read as float4): otherwise R3DG_ERR_BAD_ARG before any launch. */
int r3dg_bvh_leaf_aabbs(int P, const float* means3D, const float* scales, const float* rotations,
                        int32_t* nodes, float* aabbs, r3dg_stream_t stream);

/* Replaces create_bvh / construct_bvh (bvh/src/bvh.cu:8-27, bvh/src/construct.cu:147-266):
 * nodes / aabbs pre-filled as above are completed IN PLACE (leaf half reordered by Morton code,
 * internal nodes, parent links, subtree leaf counts, refitted boxes); morton u64[P] out.
 * tmp: r3dg_bvh_build_tmp_bytes(P) bytes of scratch. */
int r3dg_bvh_build(int P, int32_t* nodes, float* aabbs, uint64_t* morton, void* tmp, size_t tmp_bytes,
                   r3dg_stream_t stream);

/* Replaces trace_bvh_opacity (bvh/src/bvh.cu:88-116, bvh/src/trace.cu:196-287).  Ray r has
 * direction rays_d[r] and origin rays_o[r / rays_per_origin] + origin_offset * rays_d[r]
 * (rays_per_origin = 1, origin_offset = 0 reproduces the reference call; the host mirror of
 * RayTracer.trace_visibility passes the un-expanded origins and 0.05, bvh/__init__.py:63).
 * covs3D holds the INVERSE covariances [P,6].  Outputs: num_contributes i32[num_rays],
 * rendered_opacity f32[num_rays] in {0} U [0.9, 1]; every element is written.
 * tmp: r3dg_bvh_trace_tmp_bytes(P) bytes of scratch (re-packed tree). */
int r3dg_bvh_trace_opacity(int P, long long num_rays, const int32_t* nodes, const float* aabbs,
                           const float* rays_o, int rays_per_origin, float origin_offset,
                           const float* rays_d, const float* means3D, const float* covs3D,
                           const float* opacities, const float* normals, int32_t* num_contributes,
                           float* rendered_opacity, void* tmp, size_t tmp_bytes, r3dg_stream_t stream);

/* Replaces `sample_incident_rays(normals, False, N)` of the visibility bake
 * (scene/gaussian_model.py:20-28 -> utils/graphics_utils.py:9-37 fibonacci_sphere_sampling with
 * random_rotate=False -> utils/sh_utils.py:36-68 rotation_between_z; ~20 PyTorch kernels and
 * [P,N,3]-sized intermediates in the reference): dirs f32[P,N,3] unit vectors, areas f32[P,N,1]
 * = 2*pi (may be NULL).  phase f32[P] (may be NULL) = the caller's torch.rand(P) of
 * random_rotate=True (is_training): theta_i += phase[g]*2*pi.  Same op-by-op fp32 rounding as
 * the PyTorch expression. */
int r3dg_sample_incident_dirs(int P, int N, const float* normals, const float* phase, float* dirs,
                              float* areas, r3dg_stream_t stream);

/* The visibility bake of `GaussianModel.update_visibility` (scene/gaussian_model.py:312-342) for
 * the Gaussians of leaf slots [first_slot, first_slot + count) of a built tree (slot = position in
 * Morton order; 0, P bakes everything) in ONE launch: per Gaussian g and sample i the ray
 * direction is generated in the kernel exactly as r3dg_sample_incident_dirs does (never read from
 * HBM), the origin is mean_g + origin_offset * dir (0.05, bvh/__init__.py:63), and the ray is
 * traced like r3dg_bvh_trace_opacity.  Results are written to row g of the FULL-size outputs
 * visibility f32[P,N], num_contributes i32[P,N] (may be NULL), dirs f32[P,N,3] and areas
 * f32[P,N,1] (may be NULL: written once, here); rows of other slots are not touched.
 * tmp: r3dg_bvh_trace_tmp_bytes(P). */
int r3dg_bvh_bake_visibility(int P, int first_slot, int count, int N, const int32_t* nodes,
                             const float* aabbs, const float* means3D, const float* covs3D,
                             const float* opacities, const float* normals, float origin_offset,
                             int32_t* num_contributes, float* visibility, float* dirs, float* areas,
                             void* tmp, size_t tmp_bytes, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Optional fused epilogue of the rasterizer call sites (SURVEY.md §8(f)2):
 *     feature / opacity.clamp_min(1e-5) * (num_contrib > 0)
 * (gaussian_renderer/neilf.py:135-137, render.py:106-108; 3 PyTorch kernels forward, ~6 backward).
 * feature / out / dL_* are [S,HW] planar, opacity [HW], n_contrib i32[HW].
 * ------------------------------------------------------------------------------------------ */
int r3dg_unpremultiply_forward(int S, long long HW, const float* feature, const float* opacity,
                               const int32_t* n_contrib, float* out, r3dg_stream_t stream);
int r3dg_unpremultiply_backward(int S, long long HW, const float* feature, const float* opacity,
                                const int32_t* n_contrib, const float* dL_dout, float* dL_dfeature,
                                float* dL_dopacity, r3dg_stream_t stream);

/* Optional fused feature pack in front of the rasterizer (SURVEY.md §8(f)2; gaussian_renderer/neilf.py:110-126,
 * render.py:88-93): features[P,S] = cat([depths, depths^2, src_0, src_1, ...], -1) with
 * depths = (cat([means3D, 1]) @ viewmatrix)[:, 2] — means3D / viewmatrix NULL: no depth channels.  S must equal
 * (2 if depth) + sum(width).  Backward: writes every source's gradient slice contiguous (ptr NULL: skipped) and, when
 * dL_dmeans3D is given, the gradient through the two depth channels.  dL_dviewmatrix [16] (optional, NULL = none):
 * the gradient of the depth channels with respect to viewmatrix, sum_g (g_z + 2 z g_z2) [m_g,1] in elements 2, 6, 10,
 * 14 (the column that gives the depth) and exactly 0 elsewhere; summed in a fixed order through `work` (at least
 * r3dg_raster_cam_grad_bytes(P, 1) bytes) like the rasterizer's camera gradients.  dL_dviewmatrix without depth
 * channels or with too small a workspace returns R3DG_ERR_BAD_ARG. */
#define R3DG_PACK_MAX 16
typedef struct r3dg_pack_src {
    const float* ptr;              /* [P,width] contiguous (backward: destination of the gradient slice) */
    int width;
} r3dg_pack_src;
int r3dg_pack_features_forward(int P, int S, const float* means3D, const float* viewmatrix, int num,
                               const r3dg_pack_src* srcs, float* out, r3dg_stream_t stream);
int r3dg_pack_features_backward(int P, int S, const float* means3D, const float* viewmatrix,
                                const float* dL_dout, int num, const r3dg_pack_src* dsts,
                                float* dL_dmeans3D, float* dL_dviewmatrix, void* work, size_t work_bytes,
                                r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Densification surgery (SURVEY.md §8(f)3): stable compaction of the rows of MANY per-Gaussian tensors
 * by one keep-mask.  Replaces the ~40 `tensor[mask]` boolean-index launches of
 * `_prune_optimizer` / `prune_points` / `densify_and_prune` (scene/gaussian_model.py:682-729,890-929):
 *   r3dg_compact_scan  : exclusive prefix sum of keep[P] into tmp, number of kept rows -> *count_host
 *                        (pinned host int or NULL; copied asynchronously on `stream`);
 *   r3dg_compact_rows  : dst_k[offset(i)] = src_k[i] for every kept row i of every tensor k, one launch
 *                        per <= 32 tensors.  row_bytes: a multiple of 4; dst must hold count rows.
 * ------------------------------------------------------------------------------------------ */
#define R3DG_COMPACT_MAX 32
typedef struct r3dg_compact_tensor {
    const void* src;               /* [P, row_bytes] */
    void* dst;                     /* [count, row_bytes] */
    long long row_bytes;
} r3dg_compact_tensor;
size_t r3dg_compact_tmp_bytes(int P);
int r3dg_compact_scan(int P, const uint8_t* keep, void* tmp, size_t tmp_bytes, int* count_host,
                      r3dg_stream_t stream);
int r3dg_compact_rows(int P, int num_tensors, const r3dg_compact_tensor* tensors, const uint8_t* keep,
                      const void* tmp, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Stage-1 densification: `GaussianModel.add_densification_stats` and `densify_and_prune`
 * (scene/gaussian_model.py:890-937); the host side is relightable3dgaussian_b200/densify.py.
 *
 * r3dg_densify_stats: in place, for all P rows, weights_accum += weights and, where
 *   update_filter[i] != 0, xyz_gradient_accum += |viewspace_grad[i, 0:2]|, normal_gradient_accum +=
 *   |normal_grad[i]|, denom += 1, and (radii != NULL) max_radii2D = max(max_radii2D, radii).
 *   viewspace_grad rows are grad_stride floats apart (>= 2); radii and max_radii2D are both NULL or
 *   both given.  One launch, no host synchronisation.
 *
 * r3dg_densify_classify: per row, the clone / split sets and which of the row's output rows survive
 *   the final prune (the thresholds are the reference's Python floats rounded to fp32; see
 *   densify.py for their derivation), then a scan of the four output segments.  Copies 7 ints to
 *   the pinned host array `totals_host` (may be NULL) asynchronously on `stream`:
 *     [0] kept originals (segment A)  [1] kept clones (B)  [2] split rows whose copies are kept (C)
 *     [3] |S|  [4] |C|  [5] originals whose normal gradient passes the normal threshold
 *     [6] unsplit originals with weights_accum < weights_threshold
 *   The final row count is [0] + [1] + 2 [2].  3 launches (1 for P = 0).
 *
 * r3dg_densify_apply: writes every output tensor in one launch from the classify results in `tmp`
 *   and `totals` (the host copy of the 7 totals).  Output rows: kept originals, kept clones, split
 *   copy 1, split copy 2, each in row order; split copy c of the k-th split row uses
 *   samples[c |S| + k] ([2|S|,3] standard normals).  Kinds: COPY (every new row a copy), MOMENT (new
 *   rows zero), XYZ (split copies: R(q) (z * exp(s)) + x, from `rotation` [P,4] and `scaling` [P,3]),
 *   SCALING (split copies: log(exp(s) * split_recip)), ZERO (dst only: all final rows zero).
 *   At most R3DG_DENSIFY_MAX tensors; row_bytes a multiple of 4 (12 for XYZ / SCALING).  `rotation`
 *   is read as float4 and must be 16-byte aligned.
 * Bad arguments return R3DG_ERR_BAD_ARG before anything is launched.
 * ------------------------------------------------------------------------------------------ */
#define R3DG_DENSIFY_MAX 48
enum { R3DG_DENSIFY_COPY = 0, R3DG_DENSIFY_MOMENT = 1, R3DG_DENSIFY_XYZ = 2, R3DG_DENSIFY_SCALING = 3, R3DG_DENSIFY_ZERO = 4 };
typedef struct r3dg_densify_tensor {
    const void* src;               /* [P, row_bytes] (unused for ZERO) */
    void* dst;                     /* [P', row_bytes] */
    long long row_bytes;
    int kind;
} r3dg_densify_tensor;
typedef struct r3dg_densify_thresholds {
    float max_grad, max_grad_normal;   /* gradient thresholds of clone and split */
    float dense_scale;                 /* percent_dense * extent: clone if max scale <=, split if > */
    float min_opacity, weights_threshold;
    float max_screen_size;             /* used when check_size != 0 */
    float big_scale;                   /* 0.1 * extent, used when check_size != 0 */
    float split_recip;                 /* fp32 reciprocal of 0.8 * 2: split copies' scale factor */
    int check_size;
} r3dg_densify_thresholds;
int r3dg_densify_stats(int P, const float* viewspace_grad, int grad_stride, const float* normal_grad,
                       const uint8_t* update_filter, const float* weights, const int32_t* radii,
                       float* weights_accum, float* xyz_gradient_accum, float* normal_gradient_accum,
                       float* denom, float* max_radii2D, r3dg_stream_t stream);
size_t r3dg_densify_tmp_bytes(int P);
int r3dg_densify_classify(int P, const float* xyz_gradient_accum, const float* normal_gradient_accum,
                          const float* denom, const float* weights_accum, const float* scaling,
                          const float* opacity, const r3dg_densify_thresholds* thresholds, void* tmp,
                          size_t tmp_bytes, int* totals_host, r3dg_stream_t stream);
int r3dg_densify_apply(int P, const int* totals, int num_tensors, const r3dg_densify_tensor* tensors,
                       const float* rotation, const float* scaling, const float* samples, float split_recip,
                       const void* tmp, size_t tmp_bytes, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * MCMC densification (3DGS-MCMC, Kheradmand et al. 2024; gsplat's MCMCStrategy): relocation of
 * dead Gaussians onto live ones and growth under a budget, and the per-step position noise.  The
 * host side is relightable3dgaussian_b200/mcmc.py.  sigma32(l) = 1 / (1 + expf(-l)) with IEEE
 * division (torch's CUDA fp32 sigmoid).  Nothing here synchronises with the host.
 *
 * r3dg_mcmc_noise: in place, xyz += scale * sigma(-k (sigma32(l) - t)) * Sigma z per row, with
 *   Sigma = R diag(exp(s))^2 R^T, R the rotation matrix of the normalised quaternion `rotation`
 *   [P,4], s = `scaling` [P,3] (log scales), l = `opacity` [P] (logits), z [P,3] standard normals.
 *   Evaluated in fp64 from the fp32 inputs, rounded once to fp32.  1 launch (0 for P = 0).
 *
 * r3dg_mcmc_classify: row i is alive when sigma32(l_i) > min_opacity and weighs w_i = sigma32(l_i)
 *   if alive, else 0.  Writes into `tmp` the alive flags, zeroed per-row draw counts and the
 *   inclusive fp64 CDF of w, summed in a fixed order (bitwise reproducible).  3 launches.
 *
 * r3dg_mcmc_apply: draws, per-source counts, the source update and the row writes, from the
 *   classify results in `tmp`.  Draw d with uniform u_d picks the smallest i with cdf[i] >
 *   u_d * total (total = cdf[P-1]); when no row is alive every row weighs 1 (i = floor(u_d P)).
 *     n_new == 0, relocation, in place (every dst == src): uniforms [P], one per row; each dead row
 *       draws when some row is alive, and is rewritten as a copy of its source;
 *     n_new  > 0, growth (dst != src, dst holding P + n_new rows): uniforms [n_new]; output rows
 *       0..P-1 are the input rows, then one copy of the source per draw, in draw order.
 *   A source drawn c >= 1 times is corrected with N = min(c + 1, n_max) (so every copy of a source
 *   drawn more than n_max - 1 times gets the N = n_max values), o = sigma32(l) in fp64:
 *     x = 1 - (1 - o)^(1/N), coef = o / sum_{j=1..N} (-1)^(j-1) C(N,j) x^j / sqrt(j)  (fp64;
 *     coef = 1 when x = 0), l' = fp32(logit(clamp(x, min_opacity, 1 - 2^-23))),
 *     s'_k = fp32(s_k + log coef).
 *   Rewritten rows (drawn sources and their copies) take the source's row with these kinds:
 *     COPY     the source's values;      MOMENT   zero (Adam moments and the statistics);
 *     R3DG_MCMC_OPACITY (row_bytes 4)  l';  R3DG_MCMC_SCALING (row_bytes 12)  s'.
 *   Every other row keeps its values.  `opacity` / `scaling` are the same tensors the OPACITY /
 *   SCALING descriptors read.  At most R3DG_DENSIFY_MAX tensors; 2 <= n_max <= R3DG_MCMC_MAX_N;
 *   r3dg_mcmc_tmp_bytes(P, n_new) bytes of tmp (16-byte aligned) serve both phases.  3 launches.
 *   A draw never picks a dead row: where the CDF's partial sums meet it can step by one ulp, and a
 *   target inside such a step that lands on a dead row moves on to the next live row.
 * P <= 0 and every other bad argument return R3DG_ERR_BAD_ARG before anything is launched (except
 * r3dg_mcmc_noise, for which P = 0 is a no-op).
 * ------------------------------------------------------------------------------------------ */
#define R3DG_MCMC_MAX_N 64
enum { R3DG_MCMC_OPACITY = 5, R3DG_MCMC_SCALING = 6 };
size_t r3dg_mcmc_tmp_bytes(int P, int n_new);
int r3dg_mcmc_noise(int P, float* xyz, const float* rotation, const float* scaling, const float* opacity,
                    const float* z, double scale, double k, double t, r3dg_stream_t stream);
int r3dg_mcmc_classify(int P, const float* opacity, float min_opacity, void* tmp, size_t tmp_bytes,
                       r3dg_stream_t stream);
int r3dg_mcmc_apply(int P, int n_new, const float* uniforms, const float* opacity, const float* scaling,
                    double min_opacity, int n_max, int num_tensors, const r3dg_densify_tensor* tensors,
                    void* tmp, size_t tmp_bytes, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * 3D smoothing filter (Mip-Splatting's compute_3D_filter, Yu et al. 2024): the per-Gaussian
 * filter size f [P] that r3dg_raster_fwd_args.filter_3d takes, from the V training cameras.
 *   means3D [P,3]; viewmatrices [V,16] in the rasterizer's `viewmatrix` layout; intrinsics [V,6]
 *   {fx, fy, cx, cy, W, H} (device); focal_max = F, the largest fx of the V cameras (host).
 * For Gaussian i and camera c: t = [m_i, 1] V_c with z = t.z associated exactly as the
 * rasterizer's near-cull depth, u = (t.x / z) fx + cx, v = (t.y / z) fy + cy (each operation
 * rounded on its own, in that order).  The pair is valid when z > 0.2, -0.15 W <= u <= 1.15 W and
 * -0.15 H <= v <= 1.15 H, each bound the fp32 rounding of the double product.  d_i = the least z
 * of the valid pairs; a Gaussian no camera sees takes the largest d of the seen ones.  Then
 * f_i = (d_i / F) * sqrt(0.2) (fp32, in that order); f = 0 everywhere when no Gaussian is seen.
 * Differences from Mip-Splatting: each camera's own principal point (cx, cy) instead of (W/2, H/2),
 * and no 1e5 cap on d.  min and max are order-free, so the result is bitwise reproducible; nothing
 * synchronises with the host.  2 launches (0 for P = 0); tmp: r3dg_filter3d_tmp_bytes(P) bytes.
 * P < 0, V < 1 with P > 0, F not finite and positive, or a missing pointer return
 * R3DG_ERR_BAD_ARG before anything is launched.
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_filter3d_tmp_bytes(int P);
int r3dg_filter3d_compute(int P, int V, const float* means3D, const float* viewmatrices, const float* intrinsics,
                          float focal_max, float* filter_3d, void* tmp, size_t tmp_bytes, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * BRDF shading: fused `rendering_equation` (gaussian_renderer/neilf.py:339-371) + `GGX_specular`
 * (:374-406) + lat-long environment lookup (scene/direct_light_map.py:70-83) + SH incident light.
 * The reference has no extension boundary here (pure PyTorch; its render_equation.cu is dead,
 * unbuilt code with a different BRDF — SURVEY.md fact 2); the host mirror
 * relightable3dgaussian_b200/shading.py gives this entry the reference function's signature.
 * ------------------------------------------------------------------------------------------ */
typedef struct r3dg_shade_args {
    int P, N;                          /* Gaussians, incident samples per Gaussian */
    int sh_coeffs;                     /* incidents.shape[1]; 16 (degree 3) is supported */
    int env_h, env_w;                  /* environment texture size */
    const float* base_color;           /* [P,3] */
    const float* roughness;            /* [P]   */
    const float* normals;              /* [P,3] (no gradient: detached at neilf.py:94) */
    const float* viewdirs;             /* [P,3] */
    const float* incidents;            /* [P,16,3] SH coefficients of the local incident light */
    const float* env;                  /* [env_h,env_w,3] ACTIVATED environment map (softplus / HDR) */
    const float* env_transform;        /* [3,3] row-major or NULL (EnvLight.transform, envmap.py:39-42) */
    const float* visibility;           /* [P,N]   baked */
    const float* incident_dirs;        /* [P,N,3] baked */
    const float* incident_areas;       /* [P,N]   baked */
    /* forward outputs; the three [P,3] means and mean_visibility are optional (all or none),
     * the three per-sample [P,N,3] arrays are optional (all or none, eval only) */
    float* pbr;                        /* [P,3] */
    float* diffuse_light;              /* [P,3] */
    float* specular;                   /* [P,3] */
    float* mean_incident_lights;       /* [P,3] or NULL  (= incident_lights.mean(-2)) */
    float* mean_local_lights;          /* [P,3] or NULL */
    float* mean_global_lights;         /* [P,3] or NULL */
    float* mean_visibility;            /* [P]   or NULL */
    float* incident_lights;            /* [P,N,3] or NULL */
    float* local_incident_lights;      /* [P,N,3] or NULL */
    float* global_incident_lights;     /* [P,N,3] or NULL */
    /* backward: cotangents (dL_dpbr required, the others may be NULL) and gradients out */
    const float* dL_dpbr;              /* [P,3] */
    const float* dL_ddiffuse_light;    /* [P,3] or NULL */
    const float* dL_dspecular;         /* [P,3] or NULL */
    float* dL_dbase_color;             /* [P,3] */
    float* dL_droughness;              /* [P] */
    float* dL_dviewdirs;               /* [P,3] */
    float* dL_dincidents;              /* [P,16,3] */
    float* dL_denv;                    /* [env_h,env_w,3] (zeroed, then accumulated) */
    /* Several views of the same Gaussians and baked samples (V = 0 or 1: the one-view call above).
     * 1 < V <= R3DG_MAX_VIEWS: viewdirs, pbr, diffuse_light, specular, the three means, dL_dpbr, dL_ddiffuse_light,
     * dL_dspecular and dL_dviewdirs hold V blocks of the rows above ([V,P,3], mean_visibility [V,P]); dL_dbase_color,
     * dL_droughness, dL_dincidents and dL_denv are the sums over the views.  The per-sample outputs must be NULL
     * (R3DG_ERR_UNSUPPORTED).  The incident light is evaluated once per sample for all views; each view's forward
     * outputs equal a one-view call's bit for bit.  V > R3DG_MAX_VIEWS: R3DG_ERR_BAD_ARG. */
    int V;
    int transform_per_view;            /* non-zero with V > 1: env_transform is [V,3,3]; forward only (the backward
                                        * returns R3DG_ERR_UNSUPPORTED) */
    /* Deterministic mode (torch.use_deterministic_algorithms(True)): non-zero (backward only) = sums that float atomics would make
     * depend on warp arrival order are accumulated in fixed point in `det_work` (see DETERMINISTIC MODE below);
     * det_work: device workspace of at least r3dg_shade_det_bytes(env_h, env_w) bytes, zeroed by the call.  0 = the default path (det_work unused). */
    int deterministic;
    void* det_work; size_t det_work_bytes;
} r3dg_shade_args;

int r3dg_render_equation_forward(const r3dg_shade_args* args, r3dg_stream_t stream);
int r3dg_render_equation_backward(const r3dg_shade_args* args, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * DETERMINISTIC MODE.  With `deterministic` set in r3dg_raster_fwd_args, r3dg_raster_bwd_args or
 * r3dg_shade_args, the three sums that float atomics make depend on the order in which warps finish
 * are accumulated in fixed point instead (csrc/detacc.cuh): out_weights of the forward, the
 * per-Gaussian gradient rows of the backward (hence all nine rasterizer gradients) and dL_denv of the
 * shading backward.  Results are then bitwise reproducible for the same inputs on the same device,
 * whatever the scheduling (r3dg_tune knobs included).  Everything else these calls compute is already
 * order-independent and unchanged.  The fixed point is anchored to each call's cotangent scale: a
 * device reduction (no host sync) takes the largest |cotangent| m that a class of sums is linear in,
 * e = floor(log2 m) (0 for zero, NaN or Inf; |e| <= 100), and each term is rounded to a multiple of
 * 2^(e-48) (|term| < 2^(e+47); larger finite terms saturate to +-Inf, NaN / +-Inf propagate as in IEEE
 * addition); each total is rounded to fp32 once.  The classes: per view, the colour and feature slots
 * of the rasterizer's gradient rows (colour and feature cotangents) and their geometry slots (every
 * cotangent plane the compositor reads); per shading call, dL_denv (dL_dpbr, dL_ddiffuse_light,
 * dL_dspecular).  So the results are bitwise equivariant under power-of-two scaling of the cotangents,
 * and their resolution is relative to that scale, as fine at a training loss's ~2^-21 per-pixel
 * cotangents as at unit ones.  out_weights is exact (integer units of 2^-24 per pixel).
 * The workspace is the caller's, separate from `geom` (default memory use is unchanged); missing or
 * too small a workspace returns R3DG_ERR_BAD_ARG before anything is launched.
 *   r3dg_raster_fwd_det_bytes : 8 B per Gaussian;
 *   r3dg_raster_bwd_det_bytes : ~24 B per gradient-row float (8 + 4 ceil((3 + S) / 4) floats per
 *                               Gaussian): 384 MB at P = 1M, S = 5 (the per-view scale words use
 *                               the float gradient scratch of `geom`, unused in this mode);
 *   r3dg_shade_det_bytes      : ~24 B per env-texel channel + 256 B.
 * r3dg_det_sum_scaled_host: the accumulation primitive's host build (tests): *out = the sum of the n
 * host floats `terms` as the deterministic mode computes it for a class whose largest |cotangent| is
 * |anchor|.  r3dg_det_sum_host: the same with anchor 0 (e = 0).
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_raster_fwd_det_bytes(int P);
size_t r3dg_raster_bwd_det_bytes(int P, int S);
/* The deterministic workspace a backward with dL_dmeans2D_abs needs on top of r3dg_raster_bwd_det_bytes: ~48 B per
 * row (two accumulators), 48 MB at P = 1M. */
size_t r3dg_raster_bwd_det_absgrad_bytes(int P);
size_t r3dg_shade_det_bytes(int env_h, int env_w);
int r3dg_det_sum_host(long long n, const float* terms, float* out);
int r3dg_det_sum_scaled_host(long long n, const float* terms, float anchor, float* out);

/* Replaces `simple_knn._C.distCUDA2` (submodules/simple-knn/spatial.cu:15-26, simple_knn.cu:185-221):
 * mean_dist2[i] = mean of the 3 smallest squared distances from point i to the other points.
 * Init-time only in the reference (scene/gaussian_model.py:427), but imported at module import. */
size_t r3dg_knn_tmp_bytes(int P);
int r3dg_knn_dist2(int P, const float* points /* [P,3] */, float* mean_dist2 /* [P] */, void* tmp,
                   size_t tmp_bytes, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused D-SSIM loss term.  Replaces `ssim(img1, img2, window_size=11, size_average)` of
 * utils/loss_utils.py:32-63 (11x11 Gaussian window, sigma 1.5, zero padding 5, C1 = 0.01^2,
 * C2 = 0.03^2), called every step by gaussian_renderer/render.py:150 and twice by
 * gaussian_renderer/neilf.py:227,234, and as a metric by eval_nvs.py:72 and
 * eval_relighting_syn4.py:191,195.  Computed in IEEE fp32 (the reference's cuDNN convolutions
 * run in TF32 under torch's defaults); deterministic, and exactly 1 for identical images.
 * img1 / img2 / dL_dimg1 are [N,C,H,W] contiguous.
 *   r3dg_ssim_tmp_bytes : size of `tmp` for the forward (0 for an invalid shape);
 *   r3dg_ssim_forward   : out = mean of the SSIM map, [1] over everything when size_average,
 *                         else [N] per image (ssim_map.mean(1).mean(1).mean(1));
 *   r3dg_ssim_backward  : dL_dimg1 from dL_dout ([1] or [N], read on the device).  dL/dimg2 is
 *                         the same call with img1 and img2 swapped.
 * R3DG_ERR_BAD_ARG for N, C, H or W <= 0, a NULL pointer or too small a tmp;
 * R3DG_ERR_UNSUPPORTED for N*C > 65535, H*W >= 2^31 or H > 1048560.  Nothing is launched then.
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_ssim_tmp_bytes(int N, int C, int H, int W);
int r3dg_ssim_forward(int N, int C, int H, int W, const float* img1, const float* img2, int size_average,
                      float* out, void* tmp, size_t tmp_bytes, r3dg_stream_t stream);
int r3dg_ssim_backward(int N, int C, int H, int W, const float* img1, const float* img2, int size_average,
                       const float* dL_dout, float* dL_dimg1, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Fused smoothness regularisers of utils/loss_utils.py, computed in IEEE fp32 (the reference's
 * kornia convolutions run in TF32 under torch's defaults), deterministic, no float atomics.
 *
 * first_order_edge_aware_loss(data, img) (:104-105; gaussian_renderer/render.py:170,
 * gaussian_renderer/neilf.py:284,291,299):
 *   out[0] = 1/(C H W) sum_{c,y,x} sum_{d in x,y} |S_d(data_c)| * exp(-|S_d(img_c)|),
 * S_d the Sobel response divided by 8 with replicate padding of 1 (kornia spatial_gradient,
 * normalized).  data is [Cd,H,W], img [Ci,H,W], both contiguous; Cd and Ci are each 1 or
 * C = max(Cd, Ci), a 1-channel input being broadcast (torch broadcasting).
 *   r3dg_edge_aware_tmp_bytes : size of `tmp` for the forward (0 for an invalid shape);
 *   r3dg_edge_aware_backward  : dL_ddata [Cd,H,W] and / or dL_dimg [Ci,H,W] (either may be NULL,
 *                               not both) from dL_dout ([1], read on the device); a 1-channel
 *                               input's gradient is summed over the C channels.
 * R3DG_ERR_BAD_ARG for Cd, Ci, H or W <= 0, channel counts that do not broadcast, a NULL pointer
 * or too small a tmp; R3DG_ERR_UNSUPPORTED for C > 65535, H*W >= 2^31 or H > 1048560.
 *
 * tv_loss(x) (:113-117; gaussian_renderer/neilf.py:306,312), x [B,H,W] contiguous:
 *   out[0] = mean((x[:,1:,:] - x[:,:-1,:])^2) + mean((x[:,:,1:] - x[:,:,:-1])^2).
 * R3DG_ERR_BAD_ARG for B <= 0, H or W < 2 (the reference returns NaN there), a NULL pointer or
 * too small a tmp; R3DG_ERR_UNSUPPORTED for B > 65535 or H*W >= 2^31.
 *
 * The forwards launch 2 kernels, the backwards 1.  Nothing is launched on an error.
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_edge_aware_tmp_bytes(int Cd, int Ci, int H, int W);
int r3dg_edge_aware_forward(int Cd, int Ci, int H, int W, const float* data, const float* img, float* out, void* tmp,
                            size_t tmp_bytes, r3dg_stream_t stream);
int r3dg_edge_aware_backward(int Cd, int Ci, int H, int W, const float* data, const float* img, const float* dL_dout,
                             float* dL_ddata, float* dL_dimg, r3dg_stream_t stream);
size_t r3dg_tv_tmp_bytes(int B, int H, int W);
int r3dg_tv_forward(int B, int H, int W, const float* x, float* out, void* tmp, size_t tmp_bytes, r3dg_stream_t stream);
int r3dg_tv_backward(int B, int H, int W, const float* x, const float* dL_dout, float* dL_dx, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Bilateral-grid colour correction (Wang et al., SIGGRAPH 2024; gsplat's BilateralGrid / slice), a
 * per-image learnable, locally affine colour transform used during training only.
 * grids [G,12,L,GY,GX] (gsplat's layout), rgb / out / dL_dout / dL_drgb [N,3,H,W], all contiguous;
 * image_ids a DEVICE int32[N], each in [0, G) (not checked on the device: the caller validates them).
 * For pixel (px, py) of image n with colour (r, g, b):
 *   ix = (px + 0.5) (GX-1) / W, iy = (py + 0.5) (GY-1) / H, iz = (0.299 r + 0.587 g + 0.114 b) (L-1),
 *   each clamped to [0, size-1] (F.grid_sample, align_corners=True, padding_mode="border");
 *   A[12] = trilinear interpolation of grids[image_ids[n]] at (ix, iy, iz), as nested lerps
 *           v0 + t (v1 - v0), x then y then z (a constant grid gives its value exactly; the identity
 *           grid [1,0,0,0, 0,1,0,0, 0,0,1,0] returns rgb bit for bit);
 *   out_c = A[4c] r + A[4c+1] g + A[4c+2] b + A[4c+3].
 *   r3dg_bilagrid_backward: dL_drgb = A^T dL_dout + (dL/diz) (L-1) (0.299, 0.587, 0.114), the luma
 *     term 0 where the unclamped iz <= 0 or >= L-1 (torch's border rule); dL_dgrids = the sum over
 *     every pixel of every image with that id of the trilinear weight times dL/dout_c (r, g, b, 1)_j,
 *     written in full (0 for ids no image uses).  Either output may be NULL, not both; dL_dgrids
 *     needs `tmp` of r3dg_bilagrid_tmp_bytes (0 for an invalid shape): per 32x32-pixel tile one
 *     partial sub-grid.
 * Bitwise reproducible run to run, with no float atomics and no host synchronisation (so also
 * under torch.use_deterministic_algorithms).  1 launch forward; 1 backward, 2 with dL_dgrids.
 * R3DG_ERR_BAD_ARG for G, N, H or W <= 0, GX, GY or L < 2, a NULL pointer the call needs or too
 * small a tmp; R3DG_ERR_UNSUPPORTED for N > 65535, H*W >= 2^31, H or W > 2^20, GX or GY > 1024,
 * L > 16, G*12*L*GY*GX >= 2^31, or when the sub-grid one 32x32 tile touches, staged in shared
 * memory, may exceed 1024 nodes: (min(GX, floor(31 (GX-1) / W) + 3)) (min(GY, floor(31 (GY-1) / H)
 * + 3)) L > 1024.  gsplat's 16x16x8 grid fits at W, H >= 52 (5 x 5 x 8 = 200 nodes from 156 px up).
 * Nothing is launched on an error.
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_bilagrid_tmp_bytes(int G, int N, int H, int W, int GX, int GY, int L);
int r3dg_bilagrid_forward(int G, int N, int H, int W, int GX, int GY, int L, const float* grids, const int* image_ids,
                          const float* rgb, float* out, r3dg_stream_t stream);
int r3dg_bilagrid_backward(int G, int N, int H, int W, int GX, int GY, int L, const float* grids, const int* image_ids,
                           const float* rgb, const float* dL_dout, float* dL_drgb, float* dL_dgrids, void* tmp,
                           size_t tmp_bytes, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Optimiser step (SURVEY.md §8f next #3).  Replaces, for all parameter groups at once, the
 * per-group `torch.optim.Adam(l, lr=0.0, eps=1e-15).step()` of scene/gaussian_model.py:489,495-497
 * (torch 1.12.1 torch/optim/adam.py:_single_tensor_adam: no weight decay, no amsgrad, no
 * maximize — the only configuration the reference uses).  `tensors` is a HOST array; every
 * entry updates param / exp_avg / exp_avg_sq in place from grad.  `step` is the 1-based count of
 * this update for that tensor (torch increments state['step'] before using it).
 *
 * Selective step: with `row_mask` set, the tensor is n / row_elems rows of `row_elems` elements and
 * only the rows whose mask byte is nonzero are updated, with the dense step's arithmetic; every
 * other row keeps param / exp_avg / exp_avg_sq bit for bit and its gradient is not used.
 * `row_mask` NULL (a zero-filled struct) is the dense step.  R3DG_ERR_BAD_ARG when a mask is given
 * with row_elems < 1 or n not a multiple of row_elems; R3DG_ERR_UNSUPPORTED when row_elems > INT_MAX.
 * ------------------------------------------------------------------------------------------ */
typedef struct r3dg_adam_tensor {
    float* param;              /* [n] */
    const float* grad;         /* [n] */
    float* exp_avg;            /* [n] */
    float* exp_avg_sq;         /* [n] */
    long long n;
    long long step;
    double lr, beta1, beta2, eps;
    const unsigned char* row_mask;   /* [n / row_elems] device bytes, or NULL */
    long long row_elems;
} r3dg_adam_tensor;
int r3dg_adam_step(int num_tensors, const r3dg_adam_tensor* tensors, r3dg_stream_t stream);

/* Measurement hooks used by bench.py (never needed by the reference's callers).
 * r3dg_launch_count: number of this library's kernels launched so far in the process.
 * r3dg_prof_begin/end: while active, every forward/backward records CUDA events on the launching
 * stream between its stages (0 project, 1 depth sort, 2 bin count, 3 bin offsets, 4 bin scatter,
 * 5 composite fwd, 6 surface/normal, 7 composite bwd, 8 projection bwd); r3dg_prof_end sums the
 * per-stage milliseconds over the recorded calls (caller synchronises first). */
unsigned long long r3dg_launch_count(void);
int r3dg_prof_begin(int max_calls);
int r3dg_prof_end(float* stage_ms /* [9] */, int* fwd_calls, int* bwd_calls);

/* Tuning knobs (development / measurement; results are identical for every setting, only the
 * kernel variant changes).  Sets knob `key` to `value`, stores the old value in *previous (may be
 * NULL); R3DG_ERR_UNSUPPORTED for an unknown key, R3DG_ERR_BAD_ARG for an out-of-range value.
 *   "shade_group"     lanes per Gaussian in the shading kernels: 8 (default), 16, 32
 *   "shade_fwd_variant" / "shade_bwd_variant"  0 per-Gaussian SH state in registers, 1 incident
 *                     coefficients in shared memory (forward default), 2 (backward, default) +
 *                     gradient accumulators in shared memory
 *   "shade_env_mode"  env-map gradient accumulation in r3dg_render_equation_backward:
 *                     2 warp-private tagged copies, 1 shared-memory atomics (default),
 *                     0 global atomics; larger textures fall back to the lower modes
 *   "composite_bulk"  1 = per-lane cp.async.bulk record staging in the forward compositor
 *                     (an experiment; the register prefetch is the default), 0 (default)
 *   "composite_fwd_ctas" / "composite_bwd_ctas"  resident CTAs per SM of the two compositors,
 *                     enforced with dynamic shared memory; 0 (default) = whatever fits
 *                     (lower settings trade occupancy for faster heaviest warps) */
int r3dg_tune(const char* key, int value, int* previous);

/* Library identification: returns a static string such as "r3dg_b200 0.1 sm_90a". */
const char* r3dg_version(void);

#ifdef __cplusplus
}
#endif
#endif /* R3DG_B200_H_ */
