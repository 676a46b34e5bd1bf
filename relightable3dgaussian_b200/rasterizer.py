"""Host-side mirror of the reference's operator surface for the rasterizer
(gaussian_renderer/r3dg_rasterization.py:32-262): `GaussianRasterizationSettings`,
`GaussianRasterizer`, `rasterize_gaussians`, with the same field names, argument meaning, return
tuple and error behaviour, on top of this project's CUDA kernels (through `_C_raster`, our stand-in for
`r3dg_rasterization._C`).
"""
import warnings
from typing import NamedTuple

import torch
import torch.nn as nn

from . import _C_raster as _C
from . import _lib


class GaussianRasterizationSettings(NamedTuple):
    # field order == gaussian_renderer/r3dg_rasterization.py:188-204
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    cx: float
    cy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    backward_geometry: bool
    computer_pseudo_normal: bool
    debug: bool


_DEFER_COUNT = False


def set_deferred_count(enabled: bool):
    """Opt-in host run-ahead (not part of the reference surface).  The reference forward blocks on
    a D2H copy of `num_rendered` (rasterizer_impl.cu:291); by default so do we, once, after the
    whole forward is enqueued.  With deferral on, a forward that will be differentiated (some input
    requires grad) returns `num_rendered` as a `_C_raster.DeferredCount` (int()-able) that is
    resolved in backward, after the backward kernels have been enqueued, so the loss and the
    backward follow the forward on the GPU without a host round trip in between.

    It cannot fail and cannot silently truncate: the first `_C_raster._LEARN` forwards of a
    (P, W, H) shape always take the synchronous path (they learn the instance counts); afterwards the
    binning buffer holds `_C_raster._HEADROOM` x the largest count seen; a view that still
    overflows is detected in backward, which then re-runs the forward with the exact size and
    differentiates that (the cotangents autograd hands over were computed from the truncated images
    of the first attempt — one warning is issued); forwards that are not differentiated
    (`torch.no_grad()`, eval renders) always take the synchronous path."""
    global _DEFER_COUNT
    _DEFER_COUNT = bool(enabled)


_ABSGRAD = False


def set_absgrad(enabled: bool):
    """Process default of the absolute screen-space gradients (not part of the reference surface): with it on, every
    `GaussianRasterizer`, `rasterize_gaussians` and `rasterize_views` call runs as with `absgrad=True`.  Together with
    `densify.install(absgrad=True)` this gives the reference's unmodified training loop the AbsGS densification
    statistic.  `set_absgrad(False)` restores the default (off)."""
    global _ABSGRAD
    _ABSGRAD = bool(enabled)


def _absgrad_on(absgrad):
    """The call's absgrad mode: its keyword, or the process default (set_absgrad)."""
    return bool(absgrad) or _ABSGRAD


def set_ray_depth(enabled: bool):
    """Process default of the ray-depth mode (not part of the reference surface).  After `set_ray_depth(True)` every
    forward that does not ask otherwise runs as with `ray_depth=True`: `GaussianRasterizer`, `rasterize_gaussians` and
    `rasterize_views` here, and `_C_raster.rasterize_gaussians` / `rasterize_views`, which the reference's own wrapper
    (gaussian_renderer/r3dg_rasterization.py over dropin/r3dg_rasterization) calls.  The depth output, and so
    surface_xyz and the pseudo-normal, then come from per-pixel depth planes instead of the Gaussians' centre depths,
    and the reference's unmodified stage-1 loop trains its normals on the better pseudo-normal.  Each backward takes
    its forward's mode from the geometry buffer.  `set_ray_depth(False)` restores the default (off)."""
    _C.set_ray_depth(enabled)


def _ray_depth_on(ray_depth):
    """The call's ray-depth mode: its keyword, or the process default (set_ray_depth)."""
    return bool(ray_depth) or _C.ray_depth_default()


def _rd_kw(ray_depth):
    """The keyword that turns on the library's ray-depth mode, only when it is on: an off call is the call without
    the mode.  (A library backward without it takes the forward's mode from the geometry buffer.)"""
    return {"ray_depth": True} if ray_depth else {}


def _rerun_rd_kw(ray_depth):
    """The deferred-count re-run's keyword: the node's mode, explicit whenever the process default could differ from
    it (the default may have changed since the forward), and no keyword when the mode is not in use at all."""
    return {"ray_depth": bool(ray_depth)} if ray_depth or _C.ray_depth_default() else {}


def _ds_kw(depth_stats):
    """The keyword that turns on the library's depth statistics, only when they are on: an off call is the call without
    them."""
    return {"depth_stats": True} if depth_stats else {}


def _ds_bwd_kw(ctx, g_stats):
    """The backward's depth-statistics keywords: the flag and the cotangents of depth2 and median_depth (None: zeros),
    only when the node's forward had them on."""
    if not getattr(ctx, "depth_stats", False):
        return {}
    g2, gm = (tuple(g_stats) + (None, None))[:2]
    return {"depth_stats": True, "dL_dout_depth2": g2, "dL_dout_median_depth": gm}


def _stats_outputs(ctx, out):
    """The node's outputs: the reference's ten, then depth2 and median_depth when the depth statistics are on."""
    return out[:10] + (tuple(out[13:15]) if ctx.depth_stats else ())


def _set_absgrad(means2D, g_abs):
    """Adds g_abs to `means2D.absgrad` on the caller's tensor object, as autograd accumulates `.grad`: set on the first
    backward, summed with what is there on later ones (retain_graph, or a tensor used in several graphs)."""
    prev = getattr(means2D, "absgrad", None)
    means2D.absgrad = g_abs if prev is None else prev + g_abs


_EXCHANGE = None


def set_grad_exchange(exchange, campos_all=None):
    """Opt-in multi-GPU data parallelism over views (not part of the single-GPU reference surface;
    SURVEY.md §8e): the factorised exchange of the SH gradient inside `loss.backward()`.

    With a `dist.FactoredGradExchange` installed, the backward of `GaussianRasterizer` does not write
    the dense `dL_dsh` [P,M,3] at all: it writes this view's rank-1 factor [P,3], all-gathers the
    factors of the ranks' views, rebuilds mean_v(dL_dsh_v) locally and hands THAT to autograd as the
    cotangent of `shs`.  This is only valid for `shs` because the reference's render functions feed the
    rasterizer `pc.get_shs` — a view-independent (concatenation) function of the leaf parameters — so
    J^T(mean_v g_v) == mean_v(J^T g_v).  Every other cotangent (means3D, features, opacity, scales,
    rotations, ...) stays THIS VIEW's: `features` / `means3D` reach the leaves through view-dependent
    maps (depth channels, brdf_color(viewdirs): render.py:91, neilf.py:88-120), so they must be
    averaged at the leaf parameters after backward — `dist.LeafGradBucket` / `dist.average_leaf_grads`,
    skipping the SH leaves.  `campos_all` [world,3] holds the camera centres of the views the ranks
    render this step, in rank order (call again per step).  All ranks must take the same path:
    a backward that cannot use an installed exchange (debug mode, no `shs`) raises instead of silently
    skipping its collectives.  While an exchange is installed the backward is always the full one, even when no
    geometry input requires grad (the appearance-only backward is not part of the exchange).
    `set_grad_exchange(None)` turns it off."""
    global _EXCHANGE
    _EXCHANGE = None if exchange is None else (exchange, campos_all)


def _debug_call(debug, fn, args, dump, message, **kw):
    """fn(*args, **kw).  In debug mode, as in the reference, a CPU snapshot of `args` taken before the call is saved to
    `dump` if it raises, followed by the keyword arguments `kw` (e.g. `antialiasing`) as one dict."""
    if not debug:
        return fn(*args, **kw)
    saved = tuple(a.cpu().clone() if isinstance(a, torch.Tensor) else a for a in args) + (dict(kw),)
    try:
        return fn(*args, **kw)
    except Exception:
        torch.save(saved, dump)
        print(message)
        raise


def _save_forward(ctx, out, surface_grads, *tensors):
    """Keeps what the backward of a forward with outputs `out` needs: `tensors`, then with `surface_grads` the forward's
    opacity and depth images (see _surface_cotangents), and the shapes of the four image outputs (_image_cotangents)."""
    # cotangents of outputs the reference's backward ignores (num_contrib, normal, surface_xyz, weights, radii)
    # stay None instead of being materialised as zero tensors (5 fill kernels per step); the four image
    # cotangents are filled in by _image_cotangents when a loss does not touch one of them
    ctx.set_materialize_grads(False)
    ctx.out_shapes = tuple(t.shape for t in out[2:6])
    ctx.surface_grads = surface_grads
    ctx.save_for_backward(*tensors, *(out[3:5] if surface_grads else ()))


def _image_cotangents(ctx, device, *grads):
    """The cotangents of the color, opacity, depth and feature outputs, zeros for those the loss does not touch."""
    return tuple(torch.zeros(shape, dtype=torch.float32, device=device) if g is None else g
                 for g, shape in zip(grads, ctx.out_shapes))


def _surface_cotangents(ctx, g_normal, g_surface_xyz):
    """(dL_dout_normal, dL_dout_surface_xyz, out_opacity, out_depth) when the node differentiates the pseudo-normal and
    surface-xyz outputs and the loss touches one of them; None otherwise."""
    if not ctx.surface_grads or (g_normal is None and g_surface_xyz is None):
        return None
    return (g_normal, g_surface_xyz) + tuple(ctx.saved_tensors[-2:])


def _input_grads(ctx, grads, cameras):
    """The gradients of the node's inputs from the library's nine (and camera gradients, if computed).  Those of the
    three inputs `cameras` (viewmatrix, projmatrix, campos) come in their shapes: None for those that do not need
    one, and for all three when none was computed.  The last five inputs, the 3D filter (a buffer, as in
    Mip-Splatting) and the antialiasing, ray-depth, depth-statistics and absgrad flags, get None."""
    g_means2D, g_colors_precomp, g_opacities, g_means3D, g_features, g_cov3Ds, g_sh, g_scales, g_rotations = grads[:9]
    cam = (None, None, None)
    if grads[9:]:
        cam = tuple(g.reshape(t.shape) if n else None for g, t, n in zip(grads[9:], cameras, ctx.needs_input_grad[11:14]))
    return (g_means3D, g_means2D, g_features, g_sh, g_colors_precomp, g_opacities, g_scales, g_rotations, g_cov3Ds,
            None, None) + cam + (None, None, None, None, None)


# the inputs of both autograd nodes whose gradients need the geometry half of the backward: means3D, means2D, opacities,
# scales, rotations, cov3Ds_precomp, viewmatrix, projmatrix, campos (features, sh and colors_precomp are appearance)
_GEOMETRY_INPUTS = (0, 1, 5, 6, 7, 8, 11, 12, 13)


def _backward_mode(ctx):
    """Keyword arguments of the node's library backward: none (the full backward) when a geometry input needs a
    gradient or a gradient exchange is installed (set_grad_exchange), otherwise the appearance-only backward for the
    appearance inputs that need one.  Frozen geometry (means2D included) thus pays only for the gradients it uses."""
    need = ctx.needs_input_grad
    if _EXCHANGE is not None or any(need[i] for i in _GEOMETRY_INPUTS):
        return {}
    return {"geometry": False, "appearance": (need[2], need[4], need[3])}


def _aa_kw(antialiasing):
    """The keyword that turns on the library's antialiased mode, only when it is on: an off call is the call without
    the mode."""
    return {"antialiasing": True} if antialiasing else {}


def _f3d_kw(filter_3d, opacities=None):
    """The keywords that turn on the library's 3D filter, only when a filter is given; the backward also takes the
    forward's opacities."""
    if filter_3d is None:
        return {}
    return {"filter_3d": filter_3d} if opacities is None else {"filter_3d": filter_3d, "opacities": opacities}


def _absgrad_kw(ctx, kw):
    """The keyword that asks the library backward for dL_dmeans2D_abs: only when the node's absgrad mode is on, means2D
    needs a gradient and the backward runs its geometry half (`kw` from _backward_mode)."""
    return {"absgrad": True} if ctx.absgrad and ctx.needs_input_grad[1] and kw.get("geometry", True) else {}


def _forward_args(rs, means3D, features, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp):
    """The positional arguments of _C.rasterize_gaussians for the settings `rs`."""
    return (rs.bg, means3D, features, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
            rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.cx, rs.cy, rs.image_height, rs.image_width, sh,
            rs.sh_degree, rs.campos, rs.prefiltered, rs.computer_pseudo_normal, rs.debug)


class _RasterizeGaussians(torch.autograd.Function):
    """Autograd node (reference :58-185).  Inputs/outputs are the reference's; cotangents of weights / n_contrib /
    radii are ignored exactly as there (:123-124 vs :132-157), and so are those of normal / surface_xyz unless
    `surface_grads` is set.  Unlike the reference, the settings' `viewmatrix`, `projmatrix` and `campos` are inputs of
    the node as well (the same tensors, passed after the settings): they get gradients when they require them, and the
    backward computes those only then."""

    @staticmethod
    def forward(ctx, means3D, means2D, features, sh, colors_precomp, opacities, scales, rotations,
                cov3Ds_precomp, raster_settings, surface_grads, viewmatrix, projmatrix, campos, filter_3d, antialiasing,
                ray_depth, depth_stats, absgrad):
        rs = raster_settings
        out = _debug_call(rs.debug, _C.rasterize_gaussians,
                          _forward_args(rs, means3D, features, sh, colors_precomp, opacities, scales, rotations,
                                        cov3Ds_precomp),
                          "snapshot_fw.dump", "\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.",
                          _defer=not rs.debug and _DEFER_COUNT and _CALL_GRAD_MODE and any(ctx.needs_input_grad),
                          **_aa_kw(antialiasing), **_f3d_kw(filter_3d), **_rd_kw(ray_depth), **_ds_kw(depth_stats))
        ctx.raster_settings = rs
        ctx.depth_stats = depth_stats
        ctx.antialiasing = antialiasing
        ctx.ray_depth = ray_depth
        ctx.absgrad = absgrad
        ctx.means2D = means2D if absgrad else None      # the caller's tensor object: the backward sets .absgrad on it
        ctx.num_rendered = out[0]
        _save_forward(ctx, out, surface_grads, colors_precomp, means3D, features, scales, rotations, cov3Ds_precomp,
                      out[9], sh, *out[10:13], opacities, filter_3d)
        return _stats_outputs(ctx, out)

    @staticmethod
    def backward(ctx, g_num_rendered, g_num_contrib, g_color, g_opacity, g_depth, g_feature,
                 g_normal, g_surface_xyz, g_weights, g_radii, *g_stats):
        rs = ctx.raster_settings
        (colors_precomp, means3D, features, scales, rotations, cov3Ds_precomp, radii, sh,
         geomBuffer, binningBuffer, imgBuffer, opacities, filter_3d) = ctx.saved_tensors[:13]
        g_color, g_opacity, g_depth, g_feature = _image_cotangents(ctx, means3D.device, g_color, g_opacity, g_depth,
                                                                   g_feature)

        def bwd_args(geom, num_rendered, binning, img):
            return (rs.bg, means3D, features, radii, colors_precomp, scales, rotations,
                    rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix, rs.projmatrix, rs.tanfovx,
                    rs.tanfovy, g_color, g_opacity, g_depth, g_feature, sh, rs.sh_degree, rs.campos,
                    geom, num_rendered, binning, img, rs.backward_geometry, rs.debug)
        ex = None
        if _EXCHANGE is not None:
            if rs.debug or sh.numel() == 0:
                raise RuntimeError("a gradient exchange is installed (set_grad_exchange) but this backward cannot take "
                                   "part in it (debug mode or no `shs` input): every rank must run the same collectives")
            ex = _EXCHANGE
        kw = _backward_mode(ctx)
        kw.update(_aa_kw(ctx.antialiasing))
        kw.update(_absgrad_kw(ctx, kw))
        kw.update(_f3d_kw(filter_3d, opacities))
        kw.update(_rd_kw(ctx.ray_depth))
        kw.update(_ds_bwd_kw(ctx, g_stats))
        if ex is not None:
            kw["_out"] = {"sh_factor": ex[0].factor}
        if any(ctx.needs_input_grad[11:14]):         # viewmatrix, projmatrix, campos
            kw["cam_grads"] = True
        # (appearance-only: the surface outputs depend only on the geometry, their cotangents have nothing to reach)
        surface = _surface_cotangents(ctx, g_normal, g_surface_xyz) if kw.get("geometry", True) else None
        if surface is not None:
            kw["surface"] = surface + (rs.cx, rs.cy)
        grads = _debug_call(rs.debug, _C.rasterize_gaussians_backward,
                            bwd_args(geomBuffer, ctx.num_rendered, binningBuffer, imgBuffer), "snapshot_bw.dump",
                            "\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n", **kw)
        if isinstance(ctx.num_rendered, _C.DeferredCount):
            ctx.num_rendered.resolve()          # after the backward kernels are in flight
            if ctx.num_rendered.overflowed:     # rare: re-run the forward with the exact size, differentiate that
                warnings.warn(f"deferred rasterization overflowed its binning buffer ({int(ctx.num_rendered)} instances); "
                              "forward re-run inside backward (cotangents come from the truncated first attempt)")
                out = _C.rasterize_gaussians(*_forward_args(rs, means3D, features, sh, colors_precomp, opacities, scales,
                                                            rotations, cov3Ds_precomp),
                                             _min_capacity=int(ctx.num_rendered) + 4096, **_aa_kw(ctx.antialiasing),
                                             **_f3d_kw(filter_3d), **_rerun_rd_kw(ctx.ray_depth),
                                             **_ds_kw(ctx.depth_stats))
                if surface is not None:         # the adjoint of the re-run's own surface pass
                    kw["surface"] = (g_normal, g_surface_xyz, out[3], out[4], rs.cx, rs.cy)
                grads = _C.rasterize_gaussians_backward(*bwd_args(out[10], out[0], out[11], out[12]), **kw)
        if ex is not None:                      # SH gradient: gather the views' factors, rebuild the mean locally
            exchange, campos_all = ex
            exchange.gather_factors()
            g_sh_avg = exchange.rebuild_sh(means3D, campos_all, rs.sh_degree)
            grads = grads[:6] + (g_sh_avg,) + grads[7:]
        if kw.get("absgrad"):
            _set_absgrad(ctx.means2D, grads[-1])
            grads = grads[:-1]
        return _input_grads(ctx, grads, (rs.viewmatrix, rs.projmatrix, rs.campos))


def _refuse_camera_grad_with_exchange(*cameras):
    """A gradient exchange renders one view per rank; camera gradients are not part of it."""
    if _EXCHANGE is not None and torch.is_grad_enabled() and any(
            isinstance(t, torch.Tensor) and t.requires_grad for t in cameras):
        raise RuntimeError("camera gradients (a viewmatrix, projmatrix or campos that requires grad) cannot be combined "
                           "with an installed gradient exchange (set_grad_exchange)")


_CALL_GRAD_MODE = True      # grad mode of the caller (inside autograd.Function.forward it is always off)


def _refuse_surface_grads_without_normals(surface_grads, computer_pseudo_normal):
    """Without the pseudo-normal pass both outputs are zeros: there is nothing to differentiate."""
    if surface_grads and not computer_pseudo_normal:
        raise ValueError("surface_grads=True needs computer_pseudo_normal=True: without it the normal and surface_xyz "
                         "outputs are zeros and have no gradient")


def _inputs(means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, features):
    """The reference's input checks (exactly one of SHs and precomputed colours, and one of a scale/rotation pair and
    a precomputed covariance), then (features, shs, colors_precomp, scales, rotations, cov3D_precomp) with every absent
    input empty and absent features [P,0]."""
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    have_sr = scales is not None or rotations is not None
    if ((scales is None or rotations is None) and cov3D_precomp is None) or (have_sr and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    empty = torch.Tensor([])
    if features is None:
        features = torch.empty_like(means3D[..., :0])
    return (features,) + tuple(empty if t is None else t for t in (shs, colors_precomp, scales, rotations, cov3D_precomp))


def rasterize_gaussians(means3D, means2D, features, sh, colors_precomp, opacities, scales,
                        rotations, cov3Ds_precomp, raster_settings, *, surface_grads=False, antialiasing=False,
                        absgrad=False, filter_3d=None, ray_depth=False, depth_stats=False):
    """The reference's rasterize_gaussians.  With `surface_grads=True` (not part of the reference surface) the
    cotangents of the pseudo-normal (output 6) and surface_xyz (output 7) flow into the gradients of the Gaussians and,
    when `viewmatrix` requires grad, of the camera; it needs `computer_pseudo_normal`.  Off (the default), they are
    ignored as in the reference.

    When no geometry input (means3D, means2D, opacities, scales, rotations, cov3Ds_precomp and the settings' viewmatrix,
    projmatrix, campos) requires grad, the backward computes only the gradients of features, sh and colors_precomp
    that are needed (frozen-geometry training; not part of the reference surface, which always runs the full
    backward).  The cotangents of opacity, depth, normal and surface_xyz then reach nothing and are not read.

    With `antialiasing=True` (not part of the reference surface) each Gaussian's opacity is multiplied by
    rho = sqrt(max(det(cov2D) / det(cov2D + 0.3 I), 2.5e-5)) before compositing, so that the fixed 0.3 px^2 screen-space
    dilation keeps the Gaussian's integrated weight instead of spreading a sub-pixel Gaussian over a pixel at full
    opacity: a model trained with it renders consistently at other resolutions and distances.  The gradients include
    rho's dependence on the 2D covariance and so reach means3D, scales, rotations, cov3Ds_precomp and the view matrix.
    Radii, tile lists and colours are those of the default mode; the images, weights and counts differ.

    With `absgrad=True`, or after `set_absgrad(True)` (not part of the reference surface), the backward also sets
    `means2D.absgrad` [P,2] on the caller's `means2D` tensor when means2D needs a gradient: per Gaussian, the sum over
    pixels of |dL/dmean2D.x| and |dL/dmean2D.y|, each pixel's term taken before the sum, in the units of
    `means2D.grad` (AbsGS; gsplat's absgrad).  Opposite pulls then no longer cancel, so the statistic of
    densify.add_densification_stats(absgrad=True) sees Gaussians that cover high-frequency detail.  Like `.grad` it
    accumulates over backward calls; the caller resets it (`means2D.absgrad = None`).  Everything else is unchanged.

    `filter_3d` (not part of the reference surface) is Mip-Splatting's 3D smoothing filter: a [P] or [P,1] fp32 CUDA
    tensor of per-Gaussian filter sizes f, from filter3d.compute_3d_filter over the training cameras.  Each Gaussian is
    drawn with scales sqrt(s^2 + f^2) and opacity o * sqrt(prod_k s_k^2 / (s_k^2 + f^2)), so that no Gaussian gets
    finer than the finest sampling any training camera gave it; zoomed-in or higher-resolution renders then show no
    erosion or speckle.  The filter is a buffer: it gets no gradient and must not require one.  A filter of the wrong
    length (stale after densification), on the CPU, not fp32 or not contiguous, and the combination with
    cov3Ds_precomp, raise ValueError before anything runs.  filter3d.fold(scales, opacities, filter_3d) gives the
    filtered Gaussians for consumers that take no filter; they render the same images.

    With `ray_depth=True`, or after `set_ray_depth(True)` (not part of the reference surface), each Gaussian adds to the
    depth output, at each pixel, the camera z at which it peaks along that pixel's ray (RaDe-GS, PGSR) instead of its
    centre's: tz + p . (pixel - mean2D), with the per-Gaussian depth plane p = conic (T0 Sigma w_z, T1 Sigma w_z) of the
    projection's local affine approximation.  A flat Gaussian on a tilted surface then renders as a tilted plane, not a
    fronto-parallel step, so surface_xyz and the pseudo-normal (outputs 6 and 7, derived from the depth) are smooth
    inside each footprint.  The depth cotangent reaches the plane: the means, scales, rotations, cov3Ds_precomp and the
    view matrix get its gradient, and means2D.grad includes -p dL/dtz.  Every other output is unchanged.

    With `depth_stats=True` (not part of the reference surface) two more outputs follow the ten: depth2 [1,H,W], the
    sum over the composited entries of w d^2 (d the depth the call composites: the centre's tz, or the ray-depth plane),
    and median_depth [1,H,W], d of the last composited entry whose transmittance before it is > 0.5 (0 where nothing
    is composited).  With op = opacity.clamp_min(1e-5), depth2 / op - (depth / op)^2 is the per-pixel depth variance of
    the reference's `lambda_depth_var`, and opacity depth2 - depth^2 the L2 depth distortion of 2DGS and Mip-NeRF 360.
    Both have gradients (the median's through the selected entry's depth only).  Every other output is unchanged, bit
    for bit.  There is no process default."""
    global _CALL_GRAD_MODE
    rs = raster_settings
    _C._check_filter_3d(filter_3d, means3D.shape[0], cov3Ds_precomp)
    _refuse_surface_grads_without_normals(surface_grads, rs.computer_pseudo_normal)
    _refuse_camera_grad_with_exchange(rs.viewmatrix, rs.projmatrix, rs.campos)
    _CALL_GRAD_MODE = torch.is_grad_enabled()
    return _RasterizeGaussians.apply(means3D, means2D, features, sh, colors_precomp, opacities,
                                     scales, rotations, cov3Ds_precomp, raster_settings, bool(surface_grads),
                                     rs.viewmatrix, rs.projmatrix, rs.campos, filter_3d, bool(antialiasing),
                                     _ray_depth_on(ray_depth), bool(depth_stats), _absgrad_on(absgrad))


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings, surface_grads=False, antialiasing=False, absgrad=False, ray_depth=False,
                 depth_stats=False):
        """`surface_grads`, `antialiasing`, `absgrad`, `ray_depth` and `depth_stats` (not part of the reference
        surface): see rasterize_gaussians."""
        super().__init__()
        self.raster_settings = raster_settings
        self.surface_grads = surface_grads
        self.antialiasing = antialiasing
        self.absgrad = absgrad
        self.ray_depth = ray_depth
        self.depth_stats = depth_stats

    def markVisible(self, positions):
        with torch.no_grad():
            rs = self.raster_settings
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                rotations=None, cov3D_precomp=None, features=None, filter_3d=None):
        """`filter_3d` (not part of the reference surface): the model's 3D filter, see rasterize_gaussians."""
        features, shs, colors_precomp, scales, rotations, cov3D_precomp = _inputs(
            means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, features)
        return rasterize_gaussians(means3D, means2D, features, shs, colors_precomp, opacities,
                                   scales, rotations, cov3D_precomp, self.raster_settings,
                                   surface_grads=self.surface_grads, antialiasing=self.antialiasing,
                                   absgrad=self.absgrad, filter_3d=filter_3d, ray_depth=self.ray_depth,
                                   depth_stats=self.depth_stats)


_VIEWS_SHARED = ("image_height", "image_width", "sh_degree", "scale_modifier", "prefiltered", "backward_geometry",
                 "computer_pseudo_normal")


class _RasterizeViews(torch.autograd.Function):
    """Autograd node of rasterize_views: V views of one set of Gaussians in one forward and one backward call."""

    @staticmethod
    def forward(ctx, means3D, means2D, features, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                settings, surface_grads, viewmatrix, projmatrix, campos, filter_3d, antialiasing, ray_depth, depth_stats,
                absgrad):
        rs = settings[0]
        bg = torch.stack([s.bg for s in settings])
        cams = [(s.tanfovx, s.tanfovy, s.cx, s.cy) for s in settings]
        out = _C.rasterize_views(bg, means3D, features, colors_precomp, opacities, scales, rotations, rs.scale_modifier,
                                 cov3Ds_precomp, viewmatrix, projmatrix, cams, rs.image_height, rs.image_width, sh,
                                 rs.sh_degree, campos, rs.prefiltered, rs.computer_pseudo_normal, **_aa_kw(antialiasing),
                                 **_f3d_kw(filter_3d), **_rd_kw(ray_depth), **_ds_kw(depth_stats))
        ctx.meta = (rs, cams, antialiasing)
        ctx.depth_stats = depth_stats
        ctx.ray_depth = ray_depth
        ctx.absgrad = absgrad
        ctx.means2D = means2D if absgrad else None
        _save_forward(ctx, out, surface_grads, colors_precomp, means3D, features, scales, rotations, cov3Ds_precomp, sh,
                      bg, viewmatrix, projmatrix, campos, *out[10:13], filter_3d,
                      opacities if filter_3d is not None else None)
        return _stats_outputs(ctx, out)

    @staticmethod
    def backward(ctx, g_num_rendered, g_num_contrib, g_color, g_opacity, g_depth, g_feature, g_normal, g_surface_xyz,
                 g_weights, g_radii, *g_stats):
        rs, cams, antialiasing = ctx.meta
        (colors_precomp, means3D, features, scales, rotations, cov3Ds_precomp, sh, bg, viewmatrix, projmatrix, campos,
         geomBuffer, binningBuffer, imgBuffer, filter_3d, opacities) = ctx.saved_tensors[:16]
        g_color, g_opacity, g_depth, g_feature = _image_cotangents(ctx, means3D.device, g_color, g_opacity, g_depth,
                                                                   g_feature)
        kw = _backward_mode(ctx)
        kw.update(_absgrad_kw(ctx, kw))
        kw.update(_f3d_kw(filter_3d, opacities))
        kw.update(_rd_kw(ctx.ray_depth))
        kw.update(_ds_bwd_kw(ctx, g_stats))
        if kw.get("geometry", True):
            kw.update(cam_grads=any(ctx.needs_input_grad[11:14]), surface=_surface_cotangents(ctx, g_normal, g_surface_xyz))
        grads = _C.rasterize_views_backward(bg, means3D, features, colors_precomp, scales, rotations, rs.scale_modifier,
                                            cov3Ds_precomp, viewmatrix, projmatrix, cams, g_color, g_opacity, g_depth,
                                            g_feature, sh, rs.sh_degree, campos, geomBuffer, binningBuffer, imgBuffer,
                                            rs.backward_geometry, **_aa_kw(antialiasing), **kw)
        if kw.get("absgrad"):
            _set_absgrad(ctx.means2D, grads[-1])
            grads = grads[:-1]
        return _input_grads(ctx, grads, (viewmatrix, projmatrix, campos))


def rasterize_views(means3D, means2D, opacities, *, settings, shs=None, colors_precomp=None, scales=None,
                    rotations=None, cov3D_precomp=None, features=None, surface_grads=False, antialiasing=False,
                    absgrad=False, filter_3d=None, ray_depth=False, depth_stats=False):
    """Render V views of the same Gaussians in one forward and one backward call (not part of the reference surface).

    `settings` holds V `GaussianRasterizationSettings`.  They must agree on image size, `sh_degree`, `scale_modifier`,
    `prefiltered`, `backward_geometry` and `computer_pseudo_normal`; `bg`, the two matrices, `campos`, `tanfov*`, `cx`
    and `cy` may differ.  `means2D` is [V,P,3] (its gradient holds each view's screen-space gradient, the input of
    the per-view densification statistics).  `features` and `colors_precomp` are shared ([P,*]) or per view
    ([V,P,*]); each gradient comes back in the shape of its input.  Every other gradient is the sum over the views.

    Returns the ten outputs of `GaussianRasterizer.forward` with a leading V: `num_rendered` is a list of V ints,
    the images are [V,C,H,W], `weights` [V,P,1], `radii` [V,P] and `num_contrib` [V,H,W] (a view of the work buffer).
    Each view equals the one-view call with its settings.  The call always reads the counts back synchronously;
    `debug=True` and an installed gradient exchange (`set_grad_exchange`) are refused, and so are more than
    `MAX_VIEWS` views or V·P >= 2^30 rows.  `surface_grads`, `antialiasing`, `absgrad`, `filter_3d` and `ray_depth` are
    those of rasterize_gaussians and apply to every view (each view with its own depth planes); `means2D.absgrad` is
    then [V,P,2], each view's own.  With `depth_stats=True`, depth2 and median_depth [V,1,H,W] follow the ten outputs,
    as in rasterize_gaussians."""
    settings = list(settings)
    V = len(settings)
    if V < 1:
        raise ValueError("rasterize_views needs at least one view")
    if V > MAX_VIEWS:
        raise ValueError(f"rasterize_views renders at most {MAX_VIEWS} views per call (got {V})")
    for name in _VIEWS_SHARED:
        vals = {getattr(s, name) for s in settings}
        if len(vals) != 1:
            raise ValueError(f"rasterize_views: the views disagree on {name} ({sorted(vals)}); it must be shared")
    _refuse_surface_grads_without_normals(surface_grads, settings[0].computer_pseudo_normal)
    if any(s.debug for s in settings):
        raise ValueError("rasterize_views does not support debug=True; render the views one by one to debug")
    if _EXCHANGE is not None:
        raise RuntimeError("rasterize_views cannot take part in an installed gradient exchange (set_grad_exchange); "
                           "the multi-GPU path renders one view per rank")
    features, shs, colors_precomp, scales, rotations, cov3D_precomp = _inputs(
        means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, features)
    P = means3D.shape[0]
    if V * P >= 1 << 30:
        raise ValueError(f"rasterize_views: V*P = {V * P} rows exceed the limit of 2^30")
    _C._check_filter_3d(filter_3d, P, cov3D_precomp)
    if tuple(means2D.shape) != (V, P, 3):
        raise ValueError(f"rasterize_views: means2D must be [V,P,3] = {(V, P, 3)}, got {tuple(means2D.shape)}")
    for name, t in (("features", features), ("colors_precomp", colors_precomp)):
        if t.dim() == 3 and t.shape[0] != V:
            raise ValueError(f"rasterize_views: per-view {name} must have V = {V} rows, got {t.shape[0]}")
    # stacked here, outside the node, so that autograd routes each view's camera gradients to that view's tensors
    viewmatrix = torch.stack([s.viewmatrix for s in settings])
    projmatrix = torch.stack([s.projmatrix for s in settings])
    campos = torch.stack([s.campos for s in settings])
    return _RasterizeViews.apply(means3D, means2D, features, shs, colors_precomp, opacities, scales, rotations,
                                 cov3D_precomp, tuple(settings), bool(surface_grads), viewmatrix, projmatrix, campos,
                                 filter_3d, bool(antialiasing), _ray_depth_on(ray_depth), bool(depth_stats),
                                 _absgrad_on(absgrad))


MAX_VIEWS = 64          # R3DG_MAX_VIEWS (include/r3dg_b200.h)


class _Unpremultiply(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feature, opacity, num_contrib):
        S, HW = feature.shape[0], feature.shape[1] * feature.shape[2]
        f, o = _lib.f32(feature), _lib.f32(opacity)
        n = num_contrib.detach().to(torch.int32).contiguous()
        out = torch.empty_like(f)
        if S > 0 and HW > 0:
            _lib.call("r3dg_unpremultiply_forward", f.device, S, HW, f.data_ptr(), o.data_ptr(), n.data_ptr(), out.data_ptr(),
                      what="unpremultiply")
        ctx.save_for_backward(f, o, n)
        return out

    @staticmethod
    def backward(ctx, g):
        f, o, n = ctx.saved_tensors
        S, HW = f.shape[0], f.shape[1] * f.shape[2]
        g = _lib.f32(g)
        d_f, d_o = torch.empty_like(f), torch.empty_like(o)
        _lib.call("r3dg_unpremultiply_backward", f.device, S, HW, f.data_ptr(), o.data_ptr(), n.data_ptr(), g.data_ptr(),
                  d_f.data_ptr(), d_o.data_ptr(), what="unpremultiply backward")
        return d_f, d_o, None


def unpremultiply(rendered_feature, rendered_opacity, num_contrib):
    """Optional fused form (SURVEY.md §8(f)2) of the epilogue the reference's render functions apply to the
    rasterizer's feature image (gaussian_renderer/neilf.py:135-137, render.py:106-108):
        rendered_feature / rendered_opacity.clamp_min(1e-5) * (num_contrib > 0)
    one HBM pass forward and one backward instead of 3 + ~6 PyTorch kernels.  The reference's own files keep
    the PyTorch expression; callers opt in by calling this instead."""
    return _Unpremultiply.apply(rendered_feature, rendered_opacity, num_contrib)


class _PackFeatures(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, viewmatrix, *tensors):
        P = tensors[0].shape[0] if tensors else means3D.shape[0]
        dev = (tensors[0] if tensors else means3D).device
        srcs = [_lib.f32(t).view(P, -1) for t in tensors]
        depth = means3D is not None
        S = (2 if depth else 0) + sum(t.shape[1] for t in srcs)
        out = torch.empty((P, S), dtype=torch.float32, device=dev)
        m = _lib.f32(means3D) if depth else None
        v = _lib.f32(viewmatrix) if depth else None
        arr = (_lib.PackSrc * max(len(srcs), 1))()
        for k, t in enumerate(srcs):
            arr[k].ptr, arr[k].width = t.data_ptr(), t.shape[1]
        if P > 0:
            _lib.call("r3dg_pack_features_forward", dev, P, S, _lib.ptr(m), _lib.ptr(v), len(srcs), arr, out.data_ptr(),
                      what="pack_features")
        ctx.meta = (P, S, [tuple(t.shape) for t in tensors], [t.shape[1] for t in srcs], depth,
                    tuple(viewmatrix.shape) if depth else None)
        ctx.save_for_backward(*([m, v] if depth else []))
        return out

    @staticmethod
    def backward(ctx, g):
        P, S, shapes, widths, depth, v_shape = ctx.meta
        m, v = ctx.saved_tensors if depth else (None, None)
        dev = g.device
        g = _lib.f32(g)
        need = ctx.needs_input_grad
        outs = [torch.empty((P, w), dtype=torch.float32, device=dev) if need[2 + k] else None for k, w in enumerate(widths)]
        d_m = torch.empty((P, 3), dtype=torch.float32, device=dev) if depth and need[0] else None
        # dL/dviewmatrix: zeros for P = 0 (no call), otherwise every element is written
        d_v = torch.zeros((16,), dtype=torch.float32, device=dev) if depth and need[1] else None
        ws = _lib.scratch(_lib.load().r3dg_raster_cam_grad_bytes(P, 1), dev) if d_v is not None else None
        arr = (_lib.PackSrc * max(len(widths), 1))()
        for k, w in enumerate(widths):
            arr[k].ptr, arr[k].width = (outs[k].data_ptr() if outs[k] is not None else None), w
        if P > 0:
            _lib.call("r3dg_pack_features_backward", dev, P, S, _lib.ptr(m), _lib.ptr(v), g.data_ptr(), len(widths), arr,
                      _lib.ptr(d_m), _lib.ptr(d_v), _lib.ptr(ws), ws.numel() if ws is not None else 0,
                      what="pack_features backward")
        return ((d_m, d_v.view(v_shape) if d_v is not None else None) +
                tuple(o.view(s) if o is not None else None for o, s in zip(outs, shapes)))


def pack_features(tensors, means3D=None, viewmatrix=None):
    """Optional fused form (SURVEY.md §8(f)2) of the feature pack the reference's render functions build in front of
    the rasterizer (gaussian_renderer/neilf.py:110-126, render.py:88-93):
        depths = (cat([means3D, 1]) @ viewmatrix)[:, 2:3];  features = cat([depths, depths.square(), *tensors], -1)
    (without means3D / viewmatrix: a plain fused cat).  One pass forward, one backward that writes every source
    gradient contiguous.  When `viewmatrix` requires grad it gets the gradient of the depth channels,
    sum_g (g_z + 2 z g_z2) [m_g,1] in the column that gives the depth (zero elsewhere), summed in a fixed order."""
    return _PackFeatures.apply(means3D, viewmatrix, *tensors)
