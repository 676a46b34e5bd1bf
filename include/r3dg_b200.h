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
/* The geometry buffer of a ray-depth call (r3dg_raster_fwd_args.ray_depth) of V views: its records and gradient rows
 * hold 4 more floats per Gaussian and view.  V below 1 is sized as 1. */
size_t r3dg_raster_ray_depth_geom_bytes(int P, int S, int V);
/* The image buffer of a call with depth statistics (r3dg_raster_fwd_args.depth_stats) of V views: the default layout
 * followed by the per-pixel median positions and one word per view.  Always larger than
 * r3dg_raster_views_img_bytes(W, H, V); V below 1 is sized as 1. */
size_t r3dg_raster_depth_stats_img_bytes(int W, int H, int V);
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
    /* Depth statistics (optional; 0 = off, the default).  Non-zero: with d the depth each accepted entry adds to
     * out_depth (tz, or the plane depth in ray-depth mode) and w = alpha T its weight,
     *   out_depth2 [1,H,W] ([V,1,H,W]) = sum w (d d) over the accepted entries in list order, like out_depth not
     *                                    normalised and without a background term;
     *   out_median_depth [1,H,W]        = d of the last accepted entry whose transmittance before it is > 0.5 (the
     *                                    entry that takes T through 0.5, or the last accepted one if T never gets
     *                                    there), 0 where no entry is accepted.
     * The image buffer must hold r3dg_raster_depth_stats_img_bytes(W, H, V) bytes (it also keeps each pixel's median
     * entry for the backward); a smaller one, or a missing output, returns R3DG_ERR_BAD_ARG before any launch.  Every
     * other output is that of 0, bit for bit. */
    int depth_stats;
    float* out_depth2;
    float* out_median_depth;
    /* Ray-depth mode (the per-pixel Gaussian depth of RaDe-GS and PGSR).  Non-zero: each Gaussian contributes to
     * out_depth, at pixel (x, y), the camera z at which it peaks along that pixel's ray under the projection's local
     * affine approximation, d = tz + p.x (x - mean2D.x) + p.y (y - mean2D.y), instead of its centre's tz.  The depth
     * plane p = conic (T0 Sigma w_z, T1 Sigma w_z) uses the record's (dilated) conic, the rows T0, T1 of T = J W, the
     * 3D covariance Sigma (after scale_modifier and the 3D filter) and w_z = (V[2], V[6], V[10]), the view matrix's
     * camera-z column.  out_depth, out_surface_xyz and out_normal change; every other output, the tile lists and
     * radii are those of 0.  The geometry buffer must then hold r3dg_raster_ray_depth_geom_bytes(P, S, V) bytes
     * (too small returns R3DG_ERR_BAD_ARG before any launch), which is always more than
     * r3dg_raster_views_geom_bytes(P, S, V): a host can tell a buffer's mode from its size.  0 = the default path. */
    int ray_depth;
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
    /* Depth statistics: non-zero when the matching forward had them on, with the cotangents of its out_depth2 and
     * out_median_depth ([V,1,H,W], both required; zeros for an output the loss does not use).  Per pixel and entry the
     * depth cotangent w dL_ddepth becomes w (dL_ddepth + 2 d dL_ddepth2) + [the entry is the pixel's median]
     * dL_dmedian, and dL/dalpha gains d^2 dL_ddepth2.  Non-zero with an image buffer smaller than
     * r3dg_raster_depth_stats_img_bytes(W, H, V) or a missing cotangent, or a cotangent given with 0, returns
     * R3DG_ERR_BAD_ARG before any launch.  The appearance-only mode ignores all three fields. */
    int depth_stats;
    const float* dL_dout_depth2;
    const float* dL_dout_median_depth;
    /* Ray-depth mode: must equal the matching forward's (zero or non-zero).  The depth cotangent then also reaches the
     * depth plane: dL_dmeans2D gains -p dL/dtz per pixel (dL_dmeans2D_abs includes it), and dL/dp reaches the conic and,
     * through T, Sigma and w_z, dL_dmeans3D, dL_dcov3D, dL_dscales, dL_drotations and dL_dviewmatrix.  det_work must
     * hold r3dg_raster_ray_depth_bwd_det_bytes(V * P, S) bytes (plus r3dg_raster_bwd_det_absgrad_bytes(V * P) with
     * dL_dmeans2D_abs) in deterministic mode.  The appearance-only mode ignores it. */
    int ray_depth;
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
 * a multiple of 4, 16-byte aligned sections.  world <= 64.  Slice r is float4s [r c, (r + 1) c) of the section, with
 * c = ceil(n_dense / 4 / world), clipped to the section (empty for the last ranks when n_dense / 4 < world).
 * R3DG_ERR_BAD_ARG before any launch: P < 0, D outside 0..3, M outside 1..16 or below (D + 1)^2, world outside 1..64,
 * rank outside [0, world), n_dense negative or not a multiple of 4, a NULL means3D, campos, dL_dsh or factors[v]
 * with P > 0, or a NULL dense[v] with n_dense > 0. */
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
 *      | 23 median_pos i32[HW]: per pixel the 1-based list position of its median entry, 0 for none (the image
 *      buffer of a call with depth statistics only, r3dg_raster_depth_stats_img_bytes)
 *      (9, 18, 19: the copy stops at max_bytes, pass R entries' worth)
 * Returns bytes written or a negative error. */
long long r3dg_raster_debug_copy(int id, int P, int S, int W, int H, const void* geom,
                                 const void* img, const void* binning, size_t binning_bytes,
                                 void* dst, long long max_bytes, r3dg_stream_t stream);
/* The same for the buffers of a ray-depth call (r3dg_raster_fwd_args.ray_depth): the geometry buffer's regions lie at
 * the mode's offsets.  r3dg_raster_debug_copy reads buffers of the default mode only. */
long long r3dg_raster_ray_depth_debug_copy(int id, int P, int S, int W, int H, const void* geom,
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
 * Ray-traced indirect light: what each Gaussian's incident rays see of the other Gaussians,
 * and its least-squares fit into the incident-light SH `incidents` (DESIGN.md §4.25).
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_bvh_bake_radiance_tmp_bytes(int P);

/* The radiance bake of a built tree: for every Gaussian g and sample i the ray of
 * r3dg_bvh_bake_visibility (direction generated in the kernel from normals[g], origin
 * mean_g + origin_offset * dir), with the same hit rule (opacity >= 1/255, not back-facing, peak
 * t >= 0.01, alpha = opacity * exp(power)).  Hits are composited front to back in ascending
 * (t, Gaussian index):  L += T * alpha * c,  T *= 1 - alpha,  until T < 1e-4.  The payload is the
 * hit Gaussian's SH shs f32[P,M,3] of degree sh_degree (0..3, M >= (sh_degree+1)^2) in the
 * rasterizer's colour convention c = max(sum_k Y_k(v) sh_k + 0.5, 0), v = normalize(mean_hit -
 * origin).  Outputs, every element written: radiance f32[P,N,3], transmittance f32[P,N] (T when
 * the ray stopped), num_hits i32[P,N] (hits composited; may be NULL).  The result is bitwise
 * reproducible.  R3DG_ERR_BAD_ARG for a bad degree / M or a short tmp, R3DG_ERR_UNSUPPORTED for
 * N beyond the bake's sample table (N * 12 > 32 KB, as r3dg_bvh_bake_visibility).
 * tmp: r3dg_bvh_bake_radiance_tmp_bytes(P). */
int r3dg_bvh_bake_radiance(int P, int N, const int32_t* nodes, const float* aabbs, const float* means3D,
                           const float* covs3D, const float* opacities, const float* normals,
                           const float* shs, int M, int sh_degree, float origin_offset, float* radiance,
                           float* transmittance, int32_t* num_hits, void* tmp, size_t tmp_bytes,
                           r3dg_stream_t stream);

/* Per Gaussian g: c = argmin (1/N) sum_i |Y(w_i)^T c - L_i|^2 + ridge |c|^2 over SH of degree
 * `degree` (0..3), with w_i the bake's N directions around normals[g] (regenerated, not read) and
 * L_i = radiance[g,i] f32[P,N,3].  The model is the shading step's local light sum_k Y_k c_k (no
 * +0.5).  out f32[P,(degree+1)^2,3] in the layout of `get_incidents()` (dc first).  Solved in
 * fp64 (Gram matrix summed in sample order, Cholesky): deterministic.  ridge must be > 0: the
 * samples cover one hemisphere only.  R3DG_ERR_BAD_ARG for a bad degree / ridge or N == 0 with
 * P > 0, R3DG_ERR_UNSUPPORTED for N * 12 > 32 KB. */
int r3dg_fit_incident_sh(int P, int N, const float* radiance, const float* normals, int degree, float ridge,
                         float* out, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * LIGHTS: point and directional lights on top of the environment light (DESIGN.md §4.26).
 * Two operations: the shadow transmittance of every (Gaussian, light) pair through a built tree,
 * and the lights' shading terms, forward and backward, for one view or several.  The caller adds
 * the terms to the shading step's pbr, diffuse_light and specular before packing the features.
 *   Light set.  K lights, 0 <= K <= R3DG_MAX_LIGHTS.  kind i32[K] is a HOST array: 0 directional,
 *   1 point.  vec f32[K,3]: a directional light's direction TOWARDS the light (any non-zero length,
 *   normalised as F.normalize, eps 1e-12), a point light's position.  color f32[K,3]: a directional
 *   light's irradiance at normal incidence, a point light's intensity (divided by the squared
 *   distance).  vec and color are device arrays.
 *   Per Gaussian g (mean m, raw normal n) and light j:
 *     directional: l = vec_j / max(|vec_j|, 1e-12),  E = color_j
 *     point:       w = vec_j - m,  l = w / max(|w|, 1e-12),  E = color_j / max(|w|^2, 1e-8)
 *       (1e-8 = R2_MIN: a light at a Gaussian's centre stays finite; |w|^2 is ((w0 w0 + w1 w1) + w2 w2)
 *       and l, like the ray origin below, is rounded op by op, so both operations see the same bits)
 *     transport = E * T[g,j] * max(n . l, 0),  f_s = GGX_specular(V, l) of the shading step (its clamps,
 *     normal flipped towards the view), and the outputs are the sums over j in index order:
 *       diffuse_light = sum transport,  specular = sum f_s transport,
 *       pbr = sum (base_color / pi + f_s) transport.
 *   This is the shading step's one incident sample along l with area 1, visibility T, global light E
 *   and zero local light: a directional light equals rendering_equation with N = 1, incident_dirs = l,
 *   incident_areas = 1, visibility = T, zero incidents and a constant env E.
 *   Shadow T[g,j]: the ray from o = m + 0.05 l (the bake's offset, rounded op by op) along l, with
 *   t_max = +inf for a directional light and |vec_j - o| for a point light.  A Gaussian is a hit when
 *   it satisfies the bake's rule (opacity >= 1/255, not back-facing, peak t >= 0.01, power <= 0), its
 *   peak t < (1 - 1e-5) t_max (so a Gaussian whose peak is at the light, e.g. with the light at its
 *   centre, is clearly not a hit rather than a tie), and the segment [0, t_max] meets its leaf box.  T is the product of
 *   (1 - opacity exp(power)) over the hits in the bake's traversal order (far child pushed first),
 *   stopped once T < 1e-4 (T as reached).  No 0.9 threshold: shadows are continuous.  T carries no
 *   gradient.  A light at a Gaussian's centre gives l = 0 and t_max = 0 there: no hit, T = 1.
 * ------------------------------------------------------------------------------------------ */
#define R3DG_MAX_LIGHTS 32

size_t r3dg_bvh_trace_lights_tmp_bytes(int P);

/* T f32[P,K] (row at the Gaussian's index, every element written) of a tree built over the same
 * Gaussians: means3D [P,3], covs3D the INVERSE covariances [P,6], opacities [P], normals [P,3].
 * Bitwise reproducible.  R3DG_ERR_BAD_ARG before any launch for P < 0, K outside 0..R3DG_MAX_LIGHTS,
 * a kind other than 0 or 1, a NULL pointer the call needs or a tmp smaller than
 * r3dg_bvh_trace_lights_tmp_bytes(P).  P = 0 or K = 0 launches nothing. */
int r3dg_bvh_trace_lights(int P, int K, const int32_t* kind, const float* vec, const int32_t* nodes,
                          const float* aabbs, const float* means3D, const float* covs3D, const float* opacities,
                          const float* normals, float* shadows, void* tmp, size_t tmp_bytes, r3dg_stream_t stream);

/* The lights' shading terms.  1 <= V <= R3DG_MAX_VIEWS views share the Gaussians, lights and shadows:
 * viewdirs, pbr, diffuse_light, specular, their cotangents and dL_dviewdirs are [V,P,3] (view-major),
 * and each view's outputs equal a one-view call's bit for bit.
 * Forward: writes pbr, diffuse_light and specular.  Backward: from dL_dpbr (required) and
 * dL_ddiffuse_light, dL_dspecular (NULL = zero) writes every element of dL_dbase_color [P,3],
 * dL_droughness [P], dL_dviewdirs [V,P,3], dL_dmeans3D [P,3] (through l and |w| of the point
 * lights), dL_dvec [K,3] and dL_dcolor [K,3]; the per-Gaussian gradients of shared inputs are the
 * sums of the per-view gradients in view order.  Normals, shadows and kind get none.  The light
 * gradients are per-CTA partials in `work` (r3dg_shade_lights_work_bytes(P, K)) summed in block
 * order: no float atomics, every output is bitwise reproducible.  R3DG_ERR_BAD_ARG before any launch
 * for P < 0, K outside 0..R3DG_MAX_LIGHTS, a kind other than 0 or 1, V outside 1..R3DG_MAX_VIEWS, a
 * NULL pointer the call needs or a short workspace.  P = 0 or K = 0 launches no kernel and zero-fills
 * the outputs that exist. */
struct r3dg_light_args {
    int P, K, V;
    const int32_t* kind;          /* HOST [K] */
    const float* vec;             /* [K,3] */
    const float* color;           /* [K,3] */
    const float* means3D;         /* [P,3] */
    const float* base_color;      /* [P,3] */
    const float* roughness;       /* [P] */
    const float* normals;         /* [P,3] */
    const float* viewdirs;        /* [V,P,3] */
    const float* shadows;         /* [P,K] */
    float* pbr;                   /* forward: [V,P,3] */
    float* diffuse_light;         /* forward: [V,P,3] */
    float* specular;              /* forward: [V,P,3] */
    const float* dL_dpbr;         /* backward: [V,P,3] */
    const float* dL_ddiffuse_light;
    const float* dL_dspecular;
    float* dL_dbase_color;
    float* dL_droughness;
    float* dL_dviewdirs;
    float* dL_dmeans3D;
    float* dL_dvec;
    float* dL_dcolor;
    void* work;                   /* backward */
    size_t work_bytes;
};
size_t r3dg_shade_lights_work_bytes(int P, int K);
int r3dg_shade_lights_forward(const struct r3dg_light_args* args, r3dg_stream_t stream);
int r3dg_shade_lights_backward(const struct r3dg_light_args* args, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * SHAPED LIGHTS: spot and rectangular area lights with soft shadows (DESIGN.md §4.28).
 * The same two operations as LIGHTS (shadow trace, shading terms forward and backward) over a
 * set of K lights, 0 <= K <= R3DG_MAX_LIGHTS, each a spot (kind 2) or a rect (kind 3).  kind i32[K]
 * is a HOST array.  Device arrays, packed per light j:
 *   pos f32[K,3]    spot: position;  rect: centre
 *   a   f32[K,3]    spot: axis, the direction the light points (any non-zero length, normalised
 *                   with eps 1e-12);  rect: half-edge vector u
 *   b   f32[K,3]    rect: half-edge vector v;  unused by a spot
 *   color f32[K,3]  spot: intensity;  rect: radiance
 *   cone f32[K,2]   spot: (cos_inner, cos_outer);  unused by a rect
 * Unused fields are not read (they may be NULL when no light of the set reads them) and get a zero
 * gradient.  M (1..R3DG_MAX_RECT_SAMPLES) and the seed are per set.
 *   Per Gaussian g (row index g, mean m, raw normal n) and light j:
 *     spot:  w = pos - m,  l = w / max(|w|, 1e-12) (exactly a point light's l),
 *            x = clamp((-l . a^ - cos_outer) / max(cos_inner - cos_outer, 1e-6), 0, 1),
 *            E = color * x^2 (3 - 2x) / max(|w|^2, 1e-8);  one shadow ray, a point light's at pos.
 *     rect:  a one-sided parallelogram y(s,t) = pos + s u + t v, s,t in [-1,1], emitting along
 *            n_e = normalize(u x v), area A = 4 |u x v|.  M x M stratified samples (i,k),
 *            sample index q = i M + k:  s = -1 + (2i + 2 xi1) / M,  t = -1 + (2k + 2 xi2) / M
 *            (xi in [0,1) spans the whole stratum of width 2/M),
 *            y_q = (pos + s u) + t v,  w_q = y_q - m,  l_q = w_q / max(|w_q|, 1e-12),
 *            E_q = color * max(-n_e . l_q, 0) A / (M^2 max(|w_q|^2, 1e-8)).
 *            A degenerate rect (u x v = 0) contributes 0 with finite gradients.
 *     xi: h = lowbias32(lowbias32(lowbias32(seed) ^ g) ^ j) and xi1 = (lowbias32(h ^ 2q) >> 8) 2^-24,
 *         xi2 = (lowbias32(h ^ (2q + 1)) >> 8) 2^-24, with lowbias32(x): x ^= x >> 16;
 *         x *= 0x7feb352d; x ^= x >> 15; x *= 0x846ca68b; x ^= x >> 16 (u32 arithmetic).  g is
 *         the Gaussian's row, so the trace and the shading see the same points.  s, t, y, w and l
 *         are rounded op by op in that order (one IEEE op each), identically in both operations.
 *   Rays: light j owns the columns [r_j, r_j + n_j) of the shadows T f32[P,R], n_j = 1 (spot) or
 *   M^2 (rect, column r_j + q), R = sum n_j <= R3DG_MAX_SHAPED_RAYS.
 *   Outputs, summed in light order, then sample order, with transport = E T max(n . l, 0) and f_s
 *   the shading step's GGX along l (LIGHTS): diffuse_light = sum transport,
 *   specular = sum f_s transport, pbr = sum (base_color / pi + f_s) transport.
 *   Shadow T: the LIGHTS trace of a point light at the ray's target (pos, or y_q): origin
 *   o = m + 0.05 l, t_max = |target - o|, the same hit rule, margin and T < 1e-4 stop.
 *   Gradients are those of the estimator at fixed T and fixed (s,t): the rect's flow through y_q,
 *   A and n_e.  Visibility-boundary terms (T's dependence on the light) are not included.
 * ------------------------------------------------------------------------------------------ */
#define R3DG_MAX_RECT_SAMPLES 8
#define R3DG_MAX_SHAPED_RAYS 256

/* The light set and the Gaussians of both operations.  Trace reads P, K, M, seed, kind, pos, a, b,
 * means3D and normals.  Forward additionally reads V, color, cone, base_color, roughness,
 * viewdirs [V,P,3] and shadows [P,R], and writes pbr, diffuse_light, specular [V,P,3].  Backward
 * from dL_dpbr (required) and dL_ddiffuse_light, dL_dspecular (NULL = zero) writes every element of
 * dL_dbase_color [P,3], dL_droughness [P], dL_dviewdirs [V,P,3], dL_dmeans3D [P,3], dL_dpos,
 * dL_da, dL_db, dL_dcolor [K,3] and dL_dcone [K,2]; per-Gaussian gradients of shared inputs are
 * the sums of the per-view gradients in view order, and each view's outputs equal a one-view
 * call's bit for bit.  Normals, shadows, kind and seed get none.  The light gradients are per-CTA
 * partials in `work` (r3dg_shade_shaped_lights_work_bytes(P, K)) summed in block order: no float
 * atomics, every output is bitwise reproducible.  R3DG_ERR_BAD_ARG before any launch for P < 0,
 * K outside 0..R3DG_MAX_LIGHTS, a kind other than 2 or 3, M outside 1..R3DG_MAX_RECT_SAMPLES,
 * R > R3DG_MAX_SHAPED_RAYS, V outside 1..R3DG_MAX_VIEWS (shading), a NULL pointer the call needs or
 * a short workspace.  P = 0 or K = 0 launches no kernel and zero-fills the outputs that exist. */
struct r3dg_shaped_light_args {
    int P, K, V, M;
    uint32_t seed;
    const int32_t* kind;          /* HOST [K] */
    const float* pos;             /* [K,3] */
    const float* a;               /* [K,3] */
    const float* b;               /* [K,3] */
    const float* color;           /* [K,3] */
    const float* cone;            /* [K,2] */
    const float* means3D;         /* [P,3] */
    const float* base_color;      /* [P,3] */
    const float* roughness;       /* [P] */
    const float* normals;         /* [P,3] */
    const float* viewdirs;        /* [V,P,3] */
    const float* shadows;         /* [P,R] */
    float* pbr;                   /* forward: [V,P,3] */
    float* diffuse_light;         /* forward: [V,P,3] */
    float* specular;              /* forward: [V,P,3] */
    const float* dL_dpbr;         /* backward: [V,P,3] */
    const float* dL_ddiffuse_light;
    const float* dL_dspecular;
    float* dL_dbase_color;
    float* dL_droughness;
    float* dL_dviewdirs;
    float* dL_dmeans3D;
    float* dL_dpos;
    float* dL_da;
    float* dL_db;
    float* dL_dcolor;
    float* dL_dcone;
    void* work;                   /* backward */
    size_t work_bytes;
};

/* R of a set (-1 for a bad set); the trace's tmp size */
int r3dg_shaped_lights_num_rays(int K, const int32_t* kind, int M);
size_t r3dg_bvh_trace_shaped_lights_tmp_bytes(int P);

/* T f32[P,R] (row at the Gaussian's index, every element written) of a tree built over the same
 * Gaussians (args->means3D), with covs3D the INVERSE covariances [P,6] and opacities [P]. */
int r3dg_bvh_trace_shaped_lights(const struct r3dg_shaped_light_args* args, const int32_t* nodes, const float* aabbs,
                                 const float* covs3D, const float* opacities, float* shadows, void* tmp,
                                 size_t tmp_bytes, r3dg_stream_t stream);

size_t r3dg_shade_shaped_lights_work_bytes(int P, int K);
int r3dg_shade_shaped_lights_forward(const struct r3dg_shaped_light_args* args, r3dg_stream_t stream);
int r3dg_shade_shaped_lights_backward(const struct r3dg_shaped_light_args* args, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * COMPOSE: similarity transforms of Gaussian models, K objects in one launch (DESIGN.md §4.27).
 *   Objects are contiguous row ranges: offsets is a HOST int32[K+1] with 0 = o[0] <= ... <= o[K] = P
 *   (empty ranges allowed), 1 <= K <= R3DG_MAX_OBJECTS.  Object k has quat[k] (w,x,y,z), normalised
 *   by the call as build_rotation does (q^ = q / |q|), R = R(q^) in build_rotation's convention,
 *   translation t[k] and scale s[k] > 0.  For each row p of object k, on the stored parameters:
 *     xyz' = s R xyz + t,  normal' = R normal (not renormalised),  rotation' = q^ (x) rotation
 *     (the reference's quaternion_multiply order, not renormalised),  scaling' = scaling + log s,
 *     sh'_l = D^l(R) sh_l for every band l >= 1 of each SH "rest" tensor [P,(L+1)^2-1,C]
 *   where D^l is defined by  sum_m Y_lm(d) c'_m = sum_m Y_lm(R^T d) c_m  for every unit d, Y the
 *   rasterizer's real SH basis (extended to l = 4 as the reference's eval_sh).  Up to
 *   R3DG_COMPOSE_MAX_SH rest tensors per call, each with its own L (0..4; 0 = no coefficients) and
 *   C (1 or 3).  Scale does not enter the SH.  D is built per CTA in fp64 from a generated table
 *   (csrc/sh_rotation_table.cuh) and applied in fp32.
 * Forward: one launch.  Backward: one launch plus a fixed-order finish; writes every element of the
 * per-row input gradients (dL_dxyz ... dL_dsh) and the per-object pose gradients dL_dR [K,9]
 * (row-major, w.r.t. R(q^) through xyz, normal and the SH), dL_dquat [K,4] (w.r.t. q^ through
 * q^ (x) rotation only; the caller chains both through q^ = q / |q|), dL_dtranslation [K,3] and
 * dL_dscale [K] (through xyz and log s).  The pose gradients are per-CTA partials in `work`
 * (r3dg_compose_work_bytes(P, K)) summed in a fixed order: no float atomics, every output is
 * bitwise reproducible.  An object with no rows gets zero pose gradients.
 * R3DG_ERR_BAD_ARG before any launch for P < 0, K outside 1..R3DG_MAX_OBJECTS, offsets that do not
 * rise from 0 to P, n_sh outside 0..R3DG_COMPOSE_MAX_SH, L outside 0..4, C other than 1 or 3, a
 * missing pointer the call needs or a short workspace.  P = 0 launches nothing (the backward
 * zero-fills the pose gradients).
 * ------------------------------------------------------------------------------------------ */
#define R3DG_MAX_OBJECTS 64
#define R3DG_COMPOSE_MAX_SH 3

struct r3dg_compose_args {
    int P, K;
    const int32_t* offsets;       /* HOST [K+1] */
    const float* quat;            /* [K,4] */
    const float* translation;     /* [K,3] */
    const float* scale;           /* [K] */
    const float* xyz;             /* [P,3] */
    const float* normal;          /* [P,3] */
    const float* rotation;        /* [P,4] */
    const float* scaling;         /* [P,3] log-scales */
    int n_sh;
    int sh_degree[3];
    int sh_channels[3];
    const float* sh[3];           /* [P,(L+1)^2-1,C] */
    float* xyz_out;               /* forward */
    float* normal_out;
    float* rotation_out;
    float* scaling_out;
    float* sh_out[3];
    const float* dL_dxyz_out;     /* backward: cotangents of the outputs */
    const float* dL_dnormal_out;
    const float* dL_drotation_out;
    const float* dL_dscaling_out;
    const float* dL_dsh_out[3];
    float* dL_dxyz;               /* backward: gradients of the inputs */
    float* dL_dnormal;
    float* dL_drotation;
    float* dL_dscaling;
    float* dL_dsh[3];
    float* dL_dR;                 /* [K,9] */
    float* dL_dquat;              /* [K,4] */
    float* dL_dtranslation;       /* [K,3] */
    float* dL_dscale;             /* [K] */
    void* work;                   /* backward */
    size_t work_bytes;
};
size_t r3dg_compose_work_bytes(int P, int K);
int r3dg_compose_forward(const struct r3dg_compose_args* args, r3dg_stream_t stream);
int r3dg_compose_backward(const struct r3dg_compose_args* args, r3dg_stream_t stream);

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
    /* Prefiltered environment (PREFILTERED ENVIRONMENT below).  env_pyramid: NULL = the point lookup above, or the
     * r3dg_env_pyramid_build output of `env`, whose env_h x env_w level 0 equals `env`: each incident sample then reads
     * the env averaged over its own solid angle.  dL_denv_pyramid: backward workspace of r3dg_env_pyramid_floats floats,
     * required (R3DG_ERR_BAD_ARG) whenever env_pyramid is set; dL_denv is still the complete gradient of `env`. */
    const float* env_pyramid;
    float* dL_denv_pyramid;
    /* Deterministic mode (torch.use_deterministic_algorithms(True)): non-zero (backward only) = sums that float atomics would make
     * depend on warp arrival order are accumulated in fixed point in `det_work` (see DETERMINISTIC MODE below);
     * det_work: device workspace of at least r3dg_shade_det_bytes(env_h, env_w) bytes, zeroed by the call.  0 = the default path (det_work unused). */
    int deterministic;
    void* det_work; size_t det_work_bytes;
} r3dg_shade_args;

int r3dg_render_equation_forward(const r3dg_shade_args* args, r3dg_stream_t stream);
int r3dg_render_equation_backward(const r3dg_shade_args* args, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * PREFILTERED ENVIRONMENT (the shading step's filtered mode).  Each incident sample s of Gaussian g
 * stands for a solid angle Omega = incident_areas[g,s] / N (2 pi / N in the reference), yet the point
 * lookup reads one bilinear tap of the env.  With a 1024x512 or 2000x1000 HDR map and N = 64 a sample
 * covers thousands of texels, and small bright sources alias.  The filtered mode reads a lat-long mip
 * pyramid at the sample's footprint instead; directions, visibility and areas are unchanged.
 *   Pyramid.  Level 0 is the activated env [He,We,3].  Level l+1 has ceil(H_l / 2) x ceil(W_l / 2)
 *   texels, made while level l has at least 3 rows and 3 columns (at most 16 levels); an env with
 *   fewer than 3 rows or columns has level 0 only, and the mode changes nothing for it.  Every level
 *   is read on the grid of grid_sample(align_corners=True) at its own size: rows 0 and H-1 are the
 *   poles, columns 0 and W-1 the same azimuth.  Row j stands for the latitude band
 *   [(j - 1/2) dt, (j + 1/2) dt] clipped to [0, pi], dt = pi / (H-1), column i for the azimuth cell
 *   [(i - 1/2) dp, (i + 1/2) dp] modulo 2 pi, dp = 2 pi / (W-1); a texel's weight is its cell's solid
 *   angle, 2 sin(dt/2) dp sin(theta) inside and (1 - cos(dt/2)) dp at a pole (sin(theta) clamped).
 *   A coarser texel is the mean of the finer level over its cell, each finer texel weighted by the
 *   solid angle the two cells share (fp64 sums, one rounding to fp32); a pole row is the mean over
 *   its whole cap, and column W-1 repeats column 0.  So a constant env gives that constant at every
 *   level, the solid-angle-weighted mean is kept at every level, the seam columns are equal and each
 *   pole row is constant.
 *   Level of detail.  d = the sample direction after env_transform, theta = acos(d.z),
 *   Omega0 = dt0 dp0 max(sin(theta), sin(dt0 / 2)) (level 0's texel solid angle),
 *   lambda = log2(Omega / Omega0) / 2 clamped to [0, L-1], evaluated in fp32.  The lookup blends
 *   levels floor(lambda) and floor(lambda) + 1 with weights 1 - f and f (f = the fraction), each with
 *   the four bilinear taps of the point lookup at that level's size.  At lambda <= 0 the lookup is the
 *   point lookup, its taps, arithmetic and bits.  Near the poles this isotropic footprint blurs
 *   latitude more than needed (a texel is narrow in azimuth there); that is accepted.
 *   Gradients.  lambda depends only on the baked direction and area and carries none; dL/denv is the
 *   adjoint of the taps through the pyramid (the backward folds it in with 2 (L-1) gather launches and
 *   no atomics); every other gradient keeps its form.  Deterministic mode accumulates every level in
 *   fixed point: det_work needs r3dg_shade_filtered_det_bytes(env_h, env_w) bytes.
 *   Composition: one view and several views (the filtered light is evaluated once per sample for all
 *   views, per view with per-view transforms), both light kinds, every r3dg_tune shading variant
 *   (same forward bits), the per-sample outputs (they hold the filtered light).
 *   Cost: the pyramid is ~4/3 of the env; the backward workspace as much again.  The env-gradient
 *   mode is picked from the texel count of all levels (a 16x32 env stays in shared memory).
 * r3dg_env_pyramid_levels / _floats: L, and the floats of all levels (0 for a size <= 0).
 * r3dg_env_pyramid_build: pyramid = every level of env, level after level (L - 1 launches and one
 * copy); fixed order, no atomics (bitwise reproducible), no host synchronisation.  A NULL pointer or a
 * size <= 0 returns R3DG_ERR_BAD_ARG before anything is launched.
 * ------------------------------------------------------------------------------------------ */
int r3dg_env_pyramid_levels(int env_h, int env_w);
size_t r3dg_env_pyramid_floats(int env_h, int env_w);
int r3dg_env_pyramid_build(const float* env, int env_h, int env_w, float* pyramid, r3dg_stream_t stream);
size_t r3dg_shade_filtered_det_bytes(int env_h, int env_w);

/* ------------------------------------------------------------------------------------------
 * IMPORTANCE SAMPLING of the environment light (DESIGN.md §4.31).  The bake's Fibonacci directions ignore where
 * the light is and where the BRDF points; under an HDR map with a small bright source their estimate does not
 * converge to the rendering equation.  This sampler draws each shading point's N directions from three strategies
 * and weights them by the multi-sample balance heuristic, so the shading step's unchanged estimator
 * mean_i (f_d + f_s) L_i area_i (n.d_i)+ becomes an unbiased estimate of the integral.
 *   Env table (r3dg_env_sampler_build, from the ACTIVATED env [He,We,3], He, We >= 2), on the cells of the
 *   PREFILTERED ENVIRONMENT stencil: row j is the band [(j - 1/2) dt, (j + 1/2) dt] clipped to [0, pi],
 *   dt = pi / (He-1); column i < We-1 the azimuth cell [(i - 1/2) dp, (i + 1/2) dp] modulo 2 pi, dp = 2 pi / (We-1)
 *   (columns 0 and We-1 are one azimuth).  Cell weight = max(lum, 0) over the texel's 3 x 3 neighbourhood (wrapped
 *   in azimuth, clamped in latitude; lum = 0.2126 R + 0.7152 G + 0.0722 B, a non-finite lum counts as 0) times the
 *   cell's solid angle; all weights 0: the solid angles (uniform on the sphere).  The table holds the row CDF, each
 *   row's column CDF (fp64 sums in a fixed order, rounded once to fp32: bitwise reproducible, no atomics) and each
 *   cell's pdf per steradian, P(row) P(column | row) / solid angle from those rounded CDFs.  3 launches.
 *   Strategies.  Samples i < n_env are env samples, then n_ggx GGX samples, then n_cos = N - n_env - n_ggx >= 1
 *   cosine samples.  Sample k of a strategy s with n_s samples at shading point q (Gaussian row g, or pixel y W + x)
 *   uses h = lowbias32(lowbias32(lowbias32(seed) ^ q) ^ s) (s = 0 env, 1 ggx, 2 cos), h1 = lowbias32(h ^ 0),
 *   h2 = lowbias32(h ^ 1), u1 = (((2^32 k) / n_s + h1) mod 2^32 >> 8) 2^-24, u2 = ((k 0x9E3779B9 + h2) mod 2^32 >> 8)
 *   2^-24 (integer division; a rank-1 lattice rotated per point).
 *     env: row j by the row CDF (the largest j with cdf[j] <= u1), column i by row j's column CDF, remainders t1,
 *       t2; cos theta = cos lo_j + t1 (cos hi_j - cos lo_j), formed from the table's 1 - cos (rows j <= (He-1)/2) or
 *       1 + cos (the others) of the band edges, so sin theta keeps its precision at the poles; azimuth
 *       pi - (i - 1/2 + t2) dp (the lookup's column
 *       coordinate i - 1/2 + t2); the env-space direction is mapped to the world by T^T (T = env_transform, which
 *       must be orthonormal: the lookup reads T d).  pdf: that of the cell T d falls in.
 *     ggx: around Ns = n^ sign(n^.V^) (V^ = normalize(viewdir)), a2 = max(r^4, 1e-7): cos^2 theta_h =
 *       (1 - u1) / (1 + (a2 - 1) u1) (sin^2 theta_h = a2 u1 / (1 + (a2 - 1) u1)), azimuth 2 pi u2, h rotated to Ns
 *       by rotate_from_z, l = 2 (V^.h) h - V^.
 *       pdf(l) = D(h) (Ns.h) / (4 V^.h) with h = normalize(V^ + l), D = a2 / (pi ((Ns.h)^2 (a2 - 1) + 1)^2); 0 when
 *       Ns.h <= 0 or V^.h <= 0.  A sample whose own h has V^.h <= 0 gets area 0.  The BRDF is unchanged.
 *     cos: (sqrt(u1) cos 2 pi u2, sqrt(u1) sin 2 pi u2, sqrt(1 - u1)) rotated to n^ = F.normalize(normal) by
 *       rotate_from_z; pdf (n^.l)+ / pi.  It covers every direction where the integrand can be non-zero, so the
 *       estimator is unbiased for any env, filter and table.
 *   area_i = N / ((n_env p_env(d_i) + n_ggx p_ggx(d_i)) + n_cos p_cos(d_i)) (fp32), 0 when that denominator is not a
 *   positive finite number.  The env filter's footprint is area_i / N.  Directions and areas carry no gradient; with
 *   the pdf held fixed, sum_i df/p_i is an unbiased estimate of the gradient of the integral.  Every operation of
 *   the sampler is rounded on its own, so any kernel that reproduces it gets the same bits.
 * r3dg_env_sampler_floats: the table's floats, 0 for env_h or env_w < 2.
 * r3dg_env_sampler_build: R3DG_ERR_BAD_ARG for a NULL pointer or env_h, env_w < 2, R3DG_ERR_UNSUPPORTED for more
 * than 2^31 / 3 texels, before any launch.
 * r3dg_sample_importance_dirs: dirs f32[P,N,3] and areas f32[P,N] of Gaussian rows g (q = g) from normals [P,3],
 * viewdirs [P,3] and roughness [P] (read only when n_ggx > 0), a table and env_transform ([3,3] or NULL; the
 * transform the shading step will use).  R3DG_ERR_BAD_ARG before any launch for P < 0, N < 1, n_env or n_ggx < 0,
 * n_cos < 1, n_ggx > 0 without viewdirs or roughness, seed >= 2^32, or (P > 0) a NULL normals, table, dirs or
 * areas.  One launch (none for P = 0).
 * ------------------------------------------------------------------------------------------ */
size_t r3dg_env_sampler_floats(int env_h, int env_w);
int r3dg_env_sampler_build(const float* env, int env_h, int env_w, float* table, r3dg_stream_t stream);
int r3dg_sample_importance_dirs(int P, int N, const float* normals, const float* viewdirs, const float* roughness,
                                const float* table, const float* env_transform, int n_env, int n_ggx,
                                unsigned long long seed, float* dirs, float* areas, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * PIXEL SHADING: the shading step's rendering equation at every pixel of rasterized material images
 * (deferred shading, DESIGN.md §4.29), with each pixel's visibility traced through the BVH.
 *   Layout: V views (1 <= V <= R3DG_MAX_VIEWS) of planar H x W images; view v's block of a [C,H,W] image
 *   starts at v C H W.  Views share nothing but the env: each view's outputs equal a one-view call's.
 *   Pixel p of view v is valid when mask is NULL or mask[v,p] != 0; invalid pixels are traced and shaded
 *   not at all, and every output and gradient element of theirs is +0.
 *   For a valid pixel: n^ = F.normalize(normal_p) op by op, n / max(sqrt((x*x + y*y) + z*z), 1e-12).
 *   Directions d_i = rotate_from_z(n^, fib_sample(i, N)), i < N: bit for bit r3dg_sample_incident_dirs of
 *   n^ without a phase; the area of every sample is 2 pi.
 *   Trace (r3dg_bvh_trace_pixels): T[v,i,p] is what r3dg_bvh_trace_opacity returns for the ray with
 *   origin points_p, direction d_i and origin_offset 0.05 through a tree built over the P Gaussians
 *   (same hit rule, slab test and stop rule: T in {0} U [0.9, 1]).  Reads V, H, W, N, normal, points
 *   and mask; writes T f32[V,N,H,W], every element.  No gradient.  Rays are numbered in 64 bits (V H W N
 *   may exceed 2^31), the samples of a pixel adjacent and the pixels in 8 x 8 tiles.
 *   Shading (r3dg_shade_pixels_forward / _backward): the shading step's formula (r3dg_shade_args) per
 *   pixel, with viewdir = campos_v - points_p (one fp32 subtraction per component), the raw normal_p
 *   for n.d and GGX, local light max(sum_k Y_k(d_i) inc_k, 0) (zero when incidents is NULL), global light
 *   env(transform_v d_i) T[v,i,p] (the point lookup, or the filtered one at Omega = 2 pi / N with
 *   env_pyramid), and pbr, diffuse_light, specular the means over the samples; mean_visibility = mean_i
 *   T.  Each output equals r3dg_render_equation_forward of the pixel as a row (viewdirs, T and the
 *   sampler's directions and areas) bit for bit.
 *   Backward from dL_dpbr (required), dL_ddiffuse_light and dL_dspecular (NULL = zero) writes every
 *   element of dL_dbase_color [V,3,H,W], dL_droughness [V,1,H,W], dL_dincidents [V,48,H,W] (with
 *   incidents) and dL_denv [env_h,env_w,3] (summed over all views).  None to normal, points, campos or
 *   T.  dL_denv follows r3dg_shade_args: the pyramid's dL_denv_pyramid workspace with env_pyramid, and
 *   the deterministic mode's fixed-point sums in det_work (r3dg_shade_det_bytes, or
 *   r3dg_shade_filtered_det_bytes with env_pyramid), anchored to the largest cotangent of the call.
 *   Refusals before any launch: R3DG_ERR_BAD_ARG for V outside 1..R3DG_MAX_VIEWS, H, W, N, env_h or
 *   env_w < 1, a NULL pointer the call needs, transform_per_view without env_transform, a missing
 *   dL_denv_pyramid, a missing or short det_work, or a short tmp; R3DG_ERR_UNSUPPORTED for N beyond the
 *   bake's sample table (N * 12 > 32 KB) or V H W > 2^31 - 1.
 * ------------------------------------------------------------------------------------------ */
struct r3dg_pixel_args {
    int V, H, W, N;
    int env_h, env_w;
    const float* base_color;      /* [V,3,H,W] un-premultiplied */
    const float* roughness;       /* [V,1,H,W] */
    const float* normal;          /* [V,3,H,W] (no gradient) */
    const float* points;          /* [V,3,H,W] world-space surface points */
    const float* campos;          /* [V,3] camera centres */
    const float* incidents;       /* [V,48,H,W] or NULL: channel 3k + c = SH coefficient k of colour c */
    const uint8_t* mask;          /* [V,H,W] or NULL */
    const float* env;             /* [env_h,env_w,3] ACTIVATED environment map */
    const float* env_transform;   /* NULL, [3,3], or [V,3,3] with transform_per_view */
    int transform_per_view;
    const float* env_pyramid;     /* NULL or r3dg_env_pyramid_build of env */
    float* dL_denv_pyramid;       /* backward with env_pyramid: r3dg_env_pyramid_floats floats of workspace */
    const float* visibility;      /* T [V,N,H,W] */
    float* pbr;                   /* forward: [V,3,H,W] */
    float* diffuse_light;         /* forward: [V,3,H,W] */
    float* specular;              /* forward: [V,3,H,W] */
    float* mean_visibility;       /* forward: [V,1,H,W] */
    const float* dL_dpbr;         /* backward: [V,3,H,W] */
    const float* dL_ddiffuse_light;
    const float* dL_dspecular;
    float* dL_dbase_color;
    float* dL_droughness;
    float* dL_dincidents;
    float* dL_denv;
    int deterministic;
    void* det_work;
    size_t det_work_bytes;
    /* Importance sampling (IMPORTANCE SAMPLING above).  sampler_table NULL: the Fibonacci directions above, unchanged.
     * Otherwise sample i of pixel p = y W + x (q = p in every view) is the sampler's, with n_env env samples drawn under
     * sampler_transform ([3,3] or NULL; the transform the table's samples follow, which may differ from the shading's
     * env_transform), n_ggx GGX samples (they read roughness and campos; the trace reads them too) and
     * N - n_env - n_ggx >= 1 cosine samples: the trace traces those directions, and the shading uses them with their
     * areas (the filtered env's footprint is area_i / N).  mean_visibility is then mean_i T over the importance-sampled
     * directions.  T must come from r3dg_bvh_trace_pixels with the same sampler fields.  Refused (R3DG_ERR_BAD_ARG):
     * n_env or n_ggx < 0, n_cos < 1, n_ggx > 0 without roughness or campos (trace). */
    const float* sampler_table;
    int n_env, n_ggx;
    uint32_t seed;
    const float* sampler_transform;
};

size_t r3dg_bvh_trace_pixels_tmp_bytes(int P);
/* T of the valid pixels through a tree built over P Gaussians (means3D [P,3], covs3D the INVERSE
 * covariances [P,6], opacities [P], normals [P,3]); tmp: r3dg_bvh_trace_pixels_tmp_bytes(P).  P < 1:
 * R3DG_ERR_BAD_ARG (there is no tree). */
int r3dg_bvh_trace_pixels(const struct r3dg_pixel_args* args, int P, const int32_t* nodes, const float* aabbs,
                          const float* means3D, const float* covs3D, const float* opacities, const float* normals,
                          float* T, void* tmp, size_t tmp_bytes, r3dg_stream_t stream);
int r3dg_shade_pixels_forward(const struct r3dg_pixel_args* args, r3dg_stream_t stream);
int r3dg_shade_pixels_backward(const struct r3dg_pixel_args* args, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * PIXEL LIGHTS: the shadows and shading terms of a LIGHTS or a SHAPED LIGHTS set at every pixel of
 * the PIXEL SHADING layout (DESIGN.md §4.30), so a highlight or a shadow edge varies inside one
 * Gaussian's footprint.  The caller adds the terms to r3dg_shade_pixels_forward's outputs.
 *   Light set.  K lights, 0 <= K <= R3DG_MAX_LIGHTS, kind i32[K] a HOST array, all of one family:
 *   {0 directional, 1 point} (LIGHTS, R = K shadow columns) or {2 spot, 3 rect} (SHAPED LIGHTS, M and
 *   seed as there, R = sum n_j <= R3DG_MAX_SHAPED_RAYS columns in the same order).  pos [K,3] is a
 *   LIGHTS set's vec; a, b and cone are read only by a SHAPED LIGHTS set, as there.  M must lie in
 *   1..R3DG_MAX_RECT_SAMPLES for either family.
 *   Layout: V views (1 <= V <= R3DG_MAX_VIEWS) of planar H x W images, as PIXEL SHADING; pixel p = y W + x
 *   of view v is valid when mask is NULL or mask[v,p] != 0.
 *   A valid pixel is a Gaussian row of LIGHTS / SHAPED LIGHTS with: mean m = points_p, raw normal
 *   normal_p, viewdir = campos_v - points_p (one fp32 subtraction per component), shadows T[v,:,p] and
 *   row index p for the rect hash (the same for every view, so each view equals a one-view call).
 *   Trace (r3dg_bvh_trace_pixel_lights): T[v,c,p] is the LIGHTS trace of column c's ray from m = points_p
 *   (origin m + 0.05 l, t_max +inf for a directional light and |target - o| otherwise, the same hit
 *   rule, margin and T < 1e-4 stop) through a tree built over P Gaussians; a spot's column is a point
 *   light's ray.  Reads V, H, W, K, M, seed, kind, pos, a, b, points and mask; writes T f32[V,R,H,W],
 *   every element (0 for invalid pixels, which trace nothing).  Rays are numbered in 64 bits, a
 *   pixel's columns adjacent and the pixels in 8 x 8 tiles.  No gradient.
 *   Shading (r3dg_shade_pixel_lights_forward / _backward): pbr, diffuse_light and specular [V,3,H,W]
 *   are the LIGHTS / SHAPED LIGHTS outputs of the pixel as a row, bit for bit; 0 for invalid pixels.
 *   Backward from dL_dpbr (required), dL_ddiffuse_light and dL_dspecular (NULL = zero) writes every
 *   element of dL_dbase_color [V,3,H,W] and dL_droughness [V,1,H,W] (0 for invalid pixels), and the
 *   light gradients summed over the valid pixels of every view: dL_dpos and dL_dcolor [K,3] for a
 *   LIGHTS set; dL_dpos, dL_da, dL_db, dL_dcolor [K,3] and dL_dcone [K,2] for a SHAPED LIGHTS set.
 *   None to normal, points, campos or T.  The light gradients are per-CTA partials in `work`
 *   (r3dg_shade_pixel_lights_work_bytes(V, H, W, K)) summed in block order over a grid that depends
 *   on V H W only: no float atomics, every output is bitwise reproducible.
 *   Refusals before any launch: R3DG_ERR_BAD_ARG for V outside 1..R3DG_MAX_VIEWS, H or W < 1, K outside
 *   0..R3DG_MAX_LIGHTS, a kind outside 0..3 or a set that mixes the two families, M outside
 *   1..R3DG_MAX_RECT_SAMPLES, R > R3DG_MAX_SHAPED_RAYS, a NULL pointer the call needs, a short tmp or
 *   workspace, or P < 1 (trace); R3DG_ERR_UNSUPPORTED for V H W > 2^31 - 1.  K = 0 launches no kernel
 *   and zero-fills the outputs that exist.
 * ------------------------------------------------------------------------------------------ */
struct r3dg_pixel_light_args {
    int V, H, W, K, M;
    uint32_t seed;
    const int32_t* kind;          /* HOST [K] */
    const float* pos;             /* [K,3]: vec for kinds 0 and 1 */
    const float* a;               /* [K,3] (spot, rect) */
    const float* b;               /* [K,3] (rect) */
    const float* color;           /* [K,3] */
    const float* cone;            /* [K,2] (spot) */
    const float* base_color;      /* [V,3,H,W] un-premultiplied */
    const float* roughness;       /* [V,1,H,W] */
    const float* normal;          /* [V,3,H,W] (no gradient) */
    const float* points;          /* [V,3,H,W] world-space surface points */
    const float* campos;          /* [V,3] camera centres */
    const uint8_t* mask;          /* [V,H,W] or NULL */
    const float* shadows;         /* T [V,R,H,W] */
    float* pbr;                   /* forward: [V,3,H,W] */
    float* diffuse_light;         /* forward: [V,3,H,W] */
    float* specular;              /* forward: [V,3,H,W] */
    const float* dL_dpbr;         /* backward: [V,3,H,W] */
    const float* dL_ddiffuse_light;
    const float* dL_dspecular;
    float* dL_dbase_color;        /* [V,3,H,W] */
    float* dL_droughness;         /* [V,1,H,W] */
    float* dL_dpos;               /* [K,3] */
    float* dL_da;                 /* [K,3] (SHAPED LIGHTS) */
    float* dL_db;                 /* [K,3] (SHAPED LIGHTS) */
    float* dL_dcolor;             /* [K,3] */
    float* dL_dcone;              /* [K,2] (SHAPED LIGHTS) */
    void* work;                   /* backward */
    size_t work_bytes;
};

size_t r3dg_bvh_trace_pixel_lights_tmp_bytes(int P);
/* T of every pixel through a tree built over P Gaussians (means3D [P,3], covs3D the INVERSE
 * covariances [P,6], opacities [P], normals [P,3]); tmp: r3dg_bvh_trace_pixel_lights_tmp_bytes(P). */
int r3dg_bvh_trace_pixel_lights(const struct r3dg_pixel_light_args* args, int P, const int32_t* nodes,
                                const float* aabbs, const float* means3D, const float* covs3D,
                                const float* opacities, const float* normals, float* T, void* tmp,
                                size_t tmp_bytes, r3dg_stream_t stream);
size_t r3dg_shade_pixel_lights_work_bytes(int V, int H, int W, int K);
int r3dg_shade_pixel_lights_forward(const struct r3dg_pixel_light_args* args, r3dg_stream_t stream);
int r3dg_shade_pixel_lights_backward(const struct r3dg_pixel_light_args* args, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * DENOISE: a cross-bilateral a-trous wavelet filter (Dammertz et al. 2010, the spatial filter of SVGF) over
 * planar images of the PIXEL SHADING layout (DESIGN.md §4.32), for per-pixel shading at few samples.  Its
 * edge-stopping weights come from the G-buffer guides only, never from the signal, so the filter is linear
 * in the image, y = A(guides) x, and the backward is the exact transpose A^T g.
 *   Inputs: x f32[V,C,H,W], 1 <= C <= R3DG_DENOISE_MAX_CHANNELS, 1 <= V <= R3DG_MAX_VIEWS; guides of the same
 *   views and size: normal [V,3,H,W] (un-premultiplied, any length), points [V,3,H,W] (world-space surface
 *   points), mask u8[V,H,W] or NULL (pixel p of view v is valid when mask is NULL or mask[v,p] != 0) and
 *   features [V,F,H,W], 0 <= F <= R3DG_DENOISE_MAX_FEATURES (NULL when F = 0).
 *   Unit normal: n^ = n / max(sqrt((x*x + y*y) + z*z), 1e-12) (F.normalize; a zero normal stays zero).
 *   Pass k = 0 .. L-1, 1 <= L <= R3DG_DENOISE_MAX_PASSES, step s = 2^k, y_0 = x, y_L = y:
 *     y_{k+1}(p) = sum_o w(p, p + s o) y_k(p + s o) / W_k(p),  W_k(p) = sum_o w(p, p + s o),  o in {-2..2}^2
 *   (taps in row-major order of o).  For q = p + s o != p:
 *     w(p,q) = h(o_x) h(o_y) w_n w_x w_f,  h = (1, 4, 6, 4, 1) / 16,
 *     w_n = min(max(n^_p . n^_q, 0), 1)^sigma_normal,
 *     w_x = exp(-t / sigma_plane),  t = |n^_p . (x_q - x_p)| / |x_q - x_p|  (t = 0 when x_q = x_p): the sine of the
 *           offset's angle out of p's tangent plane, free of world and image scale, near 1 across a depth step,
 *     w_f = exp(-|f_p - f_q|^2 / sigma_features^2);
 *   the centre tap (o = 0) weighs exactly h(0)^2 = 9/64, so W_k(p) > 0 on every valid pixel.  Taps outside the
 *   image or on invalid pixels weigh 0 and are not read.  Invalid pixels output 0, get gradient 0, and their
 *   values of x (and of the guides) change no output bit.  The kernels evaluate w_n w_x w_f as one
 *   exp2(sigma_normal log2 c - (t / sigma_plane + |df|^2 / sigma_features^2) log2 e), without FMA contraction.
 *   Backward (the transpose): with g_L = dL_dy and g^ = g_{k+1} / W_k (the forward's 1 / W_k, kept in `work`),
 *     g_k(q) = sum_o w(q - s o, q) g^(q - s o),  dL_dx = g_0,
 *   each weight recomputed by the forward's function from the same records, so bit for bit the forward's: a
 *   gather with no atomics, bitwise reproducible.  No gradient to the guides.
 *   Work (r3dg_denoise_work_bytes): the forward packs each pixel's unit normal, validity, point and features
 *   once into float4 records (2 + ceil((F - 1) / 4) planes), stores 1 / W_k of every pass and ping-pongs
 *   through one [V,C,H,W] image; the backward reads the records and 1 / W_k a forward with the same V, H, W,
 *   C, F and L left in `work`, and uses the same image.  x must not alias y, nor dL_dy alias dL_dx.
 *   Launches: forward 1 + L, backward L.  Each view's outputs equal a one-view call's bit for bit.
 *   Refusals before any launch: R3DG_ERR_BAD_ARG for V outside 1..R3DG_MAX_VIEWS, H or W < 1, C, F or L out of
 *   range, a sigma <= 0 or not finite, a NULL pointer the call needs, or a missing or short work;
 *   R3DG_ERR_UNSUPPORTED for V H W max(C, F) >= 2^31 (the kernels index in 32 bits).
 * ------------------------------------------------------------------------------------------ */
#define R3DG_DENOISE_MAX_CHANNELS 8
#define R3DG_DENOISE_MAX_FEATURES 8
#define R3DG_DENOISE_MAX_PASSES 6
struct r3dg_denoise_args {
    int V, H, W, C, F, L;
    float sigma_normal, sigma_plane, sigma_features;
    const float* normal;          /* forward: [V,3,H,W] (no gradient) */
    const float* points;          /* forward: [V,3,H,W] world-space surface points */
    const uint8_t* mask;          /* forward: [V,H,W] or NULL */
    const float* features;        /* forward: [V,F,H,W], NULL when F = 0 */
    const float* x;               /* forward: [V,C,H,W] */
    float* y;                     /* forward: [V,C,H,W] */
    const float* dL_dy;           /* backward: [V,C,H,W] */
    float* dL_dx;                 /* backward: [V,C,H,W] */
    void* work;                   /* r3dg_denoise_work_bytes; the backward reads what the forward wrote */
    size_t work_bytes;
};

size_t r3dg_denoise_work_bytes(int V, int H, int W, int C, int F, int L);
int r3dg_denoise_forward(const struct r3dg_denoise_args* args, r3dg_stream_t stream);
int r3dg_denoise_backward(const struct r3dg_denoise_args* args, r3dg_stream_t stream);

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
/* The deterministic backward workspace of a ray-depth call: its gradient rows hold 4 more floats (~96 B per row more
 * than r3dg_raster_bwd_det_bytes). */
size_t r3dg_raster_ray_depth_bwd_det_bytes(int P, int S);
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
 * Multi-view consistency losses (PGSR, Chen et al. 2024).  Not part of the reference surface.
 * For B pairs (r, n) of V rendered views of size H x W (r = n allowed; a view may be in several pairs):
 *   depth [V,H,W] (camera z), normal [V,3,H,W] (world frame, normalised here: n_c = normalize(R_r n) with
 *   F.normalize's eps 1e-12), gray [V,H,W] (ground truth, no gradient), all contiguous fp32 on the device;
 *   viewmatrix [V,16] on the device (row-vector world -> camera, as the rasterizer's), R_r its rotation;
 *   pair_cams a HOST [B][8] of {tan_fovx, tan_fovy, cx, cy} of the reference view, then of the neighbour;
 *   fx = W / (2 tan_fovx), fy = H / (2 tan_fovy); pixel (x, y) has the ray ((x - cx)/fx, (y - cy)/fy, 1).
 *   pairs a HOST int [B][2] of (r, n).
 * Per pixel p of view r, with (R, t) the ref -> neighbour camera transform and K_r, K_n the intrinsics:
 *   geometric: X = D K_r^-1 p~ (D = depth[r](p) > 0), Y = R X + t (Y.z > 1e-6), q = pi(K_n Y) inside
 *     [0, W-1] x [0, H-1], D' = bilinear(depth[n], q) (align corners, zero padding) > 0,
 *     X' = R^T (D' K_n^-1 q~ - t) (X'.z > 1e-6), p' = pi(K_r X'), phi = |p' - p|; geo-valid if all hold and
 *     phi < pixel_noise_threshold; w = exp(-phi) (no gradient);
 *     geo[b] = sum w phi over geo-valid pixels / max(count, 1);
 *   photometric (geo-valid pixels): d = n_c . X (|d| > 1e-6), H = K_n (R + t n_c^T / d) K_r^-1; for the 49
 *     offsets k in {-3..3}^2: a_k = gray[r](p + k) (0 outside), h_k = H (p + k, 1) (h_k.z > 1e-6),
 *     b_k = bilinear(gray[n], pi(h_k)); ncc = cov(a, b) / sqrt(var(a) var(b) + 1e-8) (population moments,
 *     cov = mean(ab) - mean(a) mean(b)); c = clamp(1 - ncc, 0, 2); photo-valid if all hold and c < 0.9;
 *     photo[b] = sum w c over photo-valid pixels / max(count, 1).
 * r3dg_multiview_forward writes geo [B], photo [B] and counts int [B][2] (geo-valid, photo-valid pixels), needs
 *   `work` of r3dg_multiview_work_bytes(B, H, W) (fp64 per-CTA partials) and reduces them in a fixed order on the
 *   device: deterministic, no host synchronisation.  2 launches.
 * r3dg_multiview_backward reads dL_dgeo [B], dL_dphoto [B] and the forward's counts and writes every element of
 *   dL_ddepth [V,H,W] and dL_dnormal [V,3,H,W]: the gradients along every path of the definition (through q, the
 *   sampling location of D', D', p', n_c, d and H), the geometric term scattered into depth[n] at the four
 *   bilinear taps of q; masks, w, counts and the clamp's flat region carry none.  It recomputes the forward per
 *   pixel.  Default: float atomics into zeroed outputs (2 memsets + 1 launch).  deterministic != 0: fixed-point
 *   accumulators (detacc.cuh) in det_work of r3dg_multiview_det_bytes(V, H, W) (96 B per view pixel and 256 B),
 *   bitwise reproducible and independent of the pairs' order (memset + 3 launches: the backward runs twice, first
 *   to measure the largest |term| of dL_ddepth and of dL_dnormal).  Each of the two has its own exponent: that of
 *   the largest |dL_dgeo[b]| / max(count, 1) and |dL_dphoto[b]| / max(count, 1), raised until its largest term
 *   fits the accumulator range 2^47, so a term the default mode writes as a finite float (e.g. a normal shorter
 *   than 1e-12, whose gradient carries 1e12) is finite here too; the resolution is 2^-48 of the larger of the two.
 * R3DG_ERR_BAD_ARG for V, H or W <= 0, B outside 1..R3DG_MAX_VIEWS, a pair index outside [0, V), a
 * non-finite camera row or tan_fov <= 0, a negative or NaN threshold, a NULL pointer the call needs, or too small
 * a workspace; R3DG_ERR_UNSUPPORTED for H*W >= 2^31 or H > 1048560.  Nothing is launched on an error.
 * ------------------------------------------------------------------------------------------ */
struct r3dg_multiview_args {
    int V, H, W, B;
    const float* depth;            /* [V,H,W] */
    const float* normal;           /* [V,3,H,W] */
    const float* gray;             /* [V,H,W] */
    const float* viewmatrix;       /* [V,16], device */
    const float* pair_cams;        /* HOST [B][8] */
    const int* pairs;              /* HOST [B][2] */
    float pixel_noise_threshold;
    float* geo;                    /* forward: [B] */
    float* photo;                  /* forward: [B] */
    int* counts;                   /* forward: written [B][2]; backward: read */
    void* work;                    /* forward */
    size_t work_bytes;
    const float* dL_dgeo;          /* backward: [B] */
    const float* dL_dphoto;        /* backward: [B] */
    float* dL_ddepth;              /* backward: [V,H,W] */
    float* dL_dnormal;             /* backward: [V,3,H,W] */
    int deterministic;
    void* det_work;
    size_t det_work_bytes;
};
size_t r3dg_multiview_work_bytes(int B, int H, int W);
size_t r3dg_multiview_det_bytes(int V, int H, int W);
int r3dg_multiview_forward(const struct r3dg_multiview_args* args, r3dg_stream_t stream);
int r3dg_multiview_backward(const struct r3dg_multiview_args* args, r3dg_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * TSDF fusion and marching-cubes mesh extraction (the 2DGS / PGSR / RaDe-GS mesh recipe).  Not part of the reference
 * surface.
 * Grid: NX, NY, NZ >= 2 points, point (i, j, k) at origin + voxel_size * (i, j, k); arrays [NX,NY,NZ] with k fastest:
 *   tsdf (fp32, initialised to 1), weight (fp32, initialised to 0) and optionally color [NX,NY,NZ,3] (fp32,
 *   initialised to 0), all contiguous on the device.
 * Cameras as in the multiview block: p_cam = [x, 1] @ viewmatrix (row-vector world -> camera), fx = W / (2 tan_fovx),
 *   fy = H / (2 tan_fovy), u = fx X/Z + cx, v = fy Y/Z + cy; the pixel is the nearest one, (floor(u + 0.5),
 *   floor(v + 0.5)).
 * Integration of V views, 1 <= V <= R3DG_MAX_VIEWS, depth [V,H,W] (camera z) and optional rgb [V,3,H,W], visited in
 *   order: view v updates grid point g only if Z > 0, the pixel lies in [0, W) x [0, H), D = depth[v](pixel) is
 *   finite with 0 < D <= depth_trunc, and sdf = D - Z >= -sdf_trunc.  Then, with obs = min(1, sdf / sdf_trunc):
 *   tsdf = (tsdf w + obs) / (w + 1), color = (color w + rgb[v](pixel)) / (w + 1), w = w + 1 (Open3D's projective
 *   TSDF with unit weights).  No gradients.  One launch, one thread per grid point: each reads its tsdf / weight /
 *   color once, walks the V views in registers and stores only if a view updated it.  IEEE fp32, no atomics: the
 *   result is bitwise reproducible, and V views in one call give the bits of V one-view calls in the same order.
 *   A non-finite viewmatrix entry (read on the device) makes the comparisons fail: the view updates nothing.
 * Extraction: a cell is valid when all 8 corners have weight > 0; a corner is inside when tsdf < 0.  A grid edge gets
 *   one vertex when its end points differ in inside-ness and one of the (up to 4) cells sharing it is valid, at
 *   p0 + t (p1 - p0), t = v0 / (v0 - v1), p0 the lower-index end; its colour is the same lerp of the corner colours.
 *   Each valid cell emits the triangles of its cube index from csrc/mc_table.cuh (every ambiguous face separates its
 *   inside corners, so the mesh is crack-free; normals point from inside to outside).  Vertices are in grid-point
 *   order, then x, y, z edge order; faces in cell order, then table order: the mesh is a function of the volume.
 *   r3dg_tsdf_extract_count classifies every grid point into `work` (r3dg_tsdf_extract_work_bytes) and scans the
 *   per-block counts (2 launches), then copies the two totals to totals_host [2] (vertices, faces) and synchronises
 *   the stream: R3DG_ERR_UNSUPPORTED when either is >= 2^31.  r3dg_tsdf_extract_emit (2 launches) then writes
 *   verts [n_verts,3], vert_colors [n_verts,3] (when color is given) and faces int [n_faces,3] from that `work`; the
 *   volume must be unchanged since the count and n_verts / n_faces must be its totals.
 * R3DG_ERR_BAD_ARG for a dimension < 2 (H, W < 1), a non-finite origin, voxel_size or sdf_trunc <= 0 or non-finite,
 * depth_trunc <= 0 or NaN (+Inf is allowed), V outside 1..R3DG_MAX_VIEWS, a camera row with tan_fov <= 0 or a
 * non-finite value, rgb given without color or color without rgb, a NULL pointer the call needs, or too small a
 * workspace; R3DG_ERR_UNSUPPORTED for NX*NY*NZ >= 2^31 or H*W >= 2^31.  Nothing is launched on an error, except
 * that the count's R3DG_ERR_UNSUPPORTED for too many vertices or faces follows its own launches.
 * ------------------------------------------------------------------------------------------ */
struct r3dg_tsdf_integrate_args {
    int NX, NY, NZ;
    float origin[3];
    float voxel_size, sdf_trunc, depth_trunc;
    float* tsdf;                   /* [NX,NY,NZ] */
    float* weight;                 /* [NX,NY,NZ] */
    float* color;                  /* [NX,NY,NZ,3] or NULL */
    int V, H, W;
    const float* depth;            /* [V,H,W] */
    const float* rgb;              /* [V,3,H,W]; iff color */
    const float* viewmatrix;       /* [V,16], device */
    const float* cams;             /* HOST [V][4]: tan_fovx, tan_fovy, cx, cy */
};
struct r3dg_tsdf_extract_args {
    int NX, NY, NZ;
    float origin[3];
    float voxel_size;
    const float* tsdf;             /* [NX,NY,NZ] */
    const float* weight;           /* [NX,NY,NZ] */
    const float* color;            /* [NX,NY,NZ,3] or NULL */
    void* work;
    size_t work_bytes;
    long long* totals_host;        /* count: HOST [2], written */
    long long n_verts, n_faces;    /* emit: the totals of the count */
    float* verts;                  /* emit: [n_verts,3] */
    float* vert_colors;            /* emit: [n_verts,3]; iff color */
    int* faces;                    /* emit: [n_faces,3] */
};
size_t r3dg_tsdf_extract_work_bytes(int NX, int NY, int NZ);
int r3dg_tsdf_integrate(const struct r3dg_tsdf_integrate_args* args, r3dg_stream_t stream);
int r3dg_tsdf_extract_count(const struct r3dg_tsdf_extract_args* args, r3dg_stream_t stream);
int r3dg_tsdf_extract_emit(const struct r3dg_tsdf_extract_args* args, r3dg_stream_t stream);

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
