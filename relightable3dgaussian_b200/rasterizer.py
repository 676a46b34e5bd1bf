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
    `GaussianRasterizer`, `rasterize_gaussians` and `rasterize_views` call runs as with `absgrad=True` (see
    rasterize_gaussians).  Together with `densify.install(absgrad=True)` this gives the reference's unmodified training
    loop the AbsGS densification statistic.  `set_absgrad(False)` restores the default (off)."""
    global _ABSGRAD
    _ABSGRAD = bool(enabled)


def set_ray_depth(enabled: bool):
    """Process default of the ray-depth mode (not part of the reference surface; see rasterize_gaussians).  After
    `set_ray_depth(True)` every forward that does not ask otherwise runs as with `ray_depth=True`: `GaussianRasterizer`,
    `rasterize_gaussians` and `rasterize_views` here, and `_C_raster.rasterize_gaussians` / `rasterize_views`, which the
    reference's own wrapper (gaussian_renderer/r3dg_rasterization.py over dropin/r3dg_rasterization) calls, so the
    reference's unmodified stage-1 loop trains its normals on the better pseudo-normal.  Each backward takes its
    forward's mode from the geometry buffer.  `set_ray_depth(False)` restores the default (off)."""
    _C.set_ray_depth(enabled)


class _Modes(NamedTuple):
    """The opt-in modes of one rasterizer call (each described in rasterize_gaussians), resolved once per call by
    _modes.  A mode that is off adds no keyword to a library call: the call is exactly the call without that mode."""
    surface_grads: bool
    antialiasing: bool
    filter_3d: object           # [P] fp32 CUDA tensor, or None
    ray_depth: bool
    depth_stats: bool
    absgrad: bool

    def forward_kw(self, rerun=False):
        """The library forward's keywords.  The deferred-count re-run (`rerun`) passes `ray_depth` explicitly whenever
        the process default could differ from the node's mode (the default may have changed since the forward)."""
        kw = {}
        if self.antialiasing:
            kw["antialiasing"] = True
        if self.filter_3d is not None:
            kw["filter_3d"] = self.filter_3d
        if self.ray_depth or (rerun and _C.ray_depth_default()):
            kw["ray_depth"] = self.ray_depth
        if self.depth_stats:
            kw["depth_stats"] = True
        return kw

    def backward_kw(self, opacities, means2D_grad, g_stats):
        """The library backward's keywords.  The filter takes the forward's `opacities` along; absgrad is asked for only
        when `means2D_grad` (means2D needs a gradient and the backward runs its geometry half); the depth statistics
        take the cotangents `g_stats` of depth2 and median_depth (None: zeros)."""
        kw = {}
        if self.antialiasing:
            kw["antialiasing"] = True
        if self.absgrad and means2D_grad:
            kw["absgrad"] = True
        if self.filter_3d is not None:
            kw.update(filter_3d=self.filter_3d, opacities=opacities)
        if self.ray_depth:
            kw["ray_depth"] = True
        if self.depth_stats:
            g2, gm = (tuple(g_stats) + (None, None))[:2]
            kw.update(depth_stats=True, dL_dout_depth2=g2, dL_dout_median_depth=gm)
        return kw


def _modes(P, cov3Ds_precomp, computer_pseudo_normal, surface_grads, antialiasing, filter_3d, ray_depth, depth_stats,
           absgrad):
    """The call's mode record: the keywords, with the process defaults of absgrad and ray_depth (set_absgrad,
    set_ray_depth).  Refuses a 3D filter the library would refuse, and surface gradients without the pseudo-normal pass
    (both outputs are then zeros: there is nothing to differentiate)."""
    _C._check_filter_3d(filter_3d, P, cov3Ds_precomp)
    if surface_grads and not computer_pseudo_normal:
        raise ValueError("surface_grads=True needs computer_pseudo_normal=True: without it the normal and surface_xyz "
                         "outputs are zeros and have no gradient")
    return _Modes(bool(surface_grads), bool(antialiasing), filter_3d, bool(ray_depth) or _C.ray_depth_default(),
                  bool(depth_stats), bool(absgrad) or _ABSGRAD)


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


# the node's tensor inputs; the settings, the mode record and the deferred-count decision follow them
_INPUTS = ("means3D", "means2D", "features", "sh", "colors_precomp", "opacities", "scales", "rotations",
           "cov3Ds_precomp", "viewmatrix", "projmatrix", "campos")
_CAMERAS = _INPUTS[_INPUTS.index("viewmatrix"):]
# the inputs whose gradients need the geometry half of the backward (the others are appearance)
_GEOMETRY = tuple(n for n in _INPUTS if n not in ("features", "sh", "colors_precomp"))
# what the node saves for its backward, followed by the forward's opacity and depth images with surface_grads; the
# work buffers stay at positions 8-10, where introspection code (debug_intermediate callers) finds them
_SAVED = ("colors_precomp", "means3D", "features", "scales", "rotations", "cov3Ds_precomp", "radii", "sh", "geomBuffer",
          "binningBuffer", "imgBuffer", "opacities", "filter_3d", "viewmatrix", "projmatrix", "campos")
# the inputs of the library backward's nine gradients, in its order (rasterize_points.cu:143-235); cameras follow
_LIB_GRADS = ("means2D", "colors_precomp", "opacities", "means3D", "features", "cov3Ds_precomp", "sh", "scales",
              "rotations")


def _forward_args(rs, x):
    """The positional arguments of _C.rasterize_gaussians for the settings `rs` and the node's inputs `x` (by name)."""
    return (rs.bg, x["means3D"], x["features"], x["colors_precomp"], x["opacities"], x["scales"], x["rotations"],
            rs.scale_modifier, x["cov3Ds_precomp"], rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.cx, rs.cy,
            rs.image_height, rs.image_width, x["sh"], rs.sh_degree, rs.campos, rs.prefiltered,
            rs.computer_pseudo_normal, rs.debug)



class _Rasterize(torch.autograd.Function):
    """Autograd node of rasterize_gaussians (reference :58-185) and rasterize_views.  One view: the settings and
    cameras [4,4], [4,4], [3] of one view; V views: V settings and the stacked cameras [V,4,4], [V,4,4], [V,3].
    Inputs/outputs are the reference's; cotangents of weights / n_contrib / radii are ignored exactly as there
    (:123-124 vs :132-157), and so are those of normal / surface_xyz unless `surface_grads` is set.  Unlike the
    reference, the cameras are inputs of the node as well: they get gradients when they require them, and the backward
    computes those only then."""

    @staticmethod
    def forward(ctx, means3D, means2D, features, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                viewmatrix, projmatrix, campos, settings, modes, defer):
        x = dict(zip(_INPUTS, (means3D, means2D, features, sh, colors_precomp, opacities, scales, rotations,
                               cov3Ds_precomp, viewmatrix, projmatrix, campos)))
        ctx.settings, ctx.modes = settings, modes
        if viewmatrix.dim() == 3:           # V views: the stacked backgrounds and the camera table
            rs = settings[0]
            ctx.views = (torch.stack([s.bg for s in settings]), [(s.tanfovx, s.tanfovy, s.cx, s.cy) for s in settings])
            out = _C.rasterize_views(ctx.views[0], means3D, features, colors_precomp, opacities, scales, rotations,
                                     rs.scale_modifier, cov3Ds_precomp, viewmatrix, projmatrix, ctx.views[1],
                                     rs.image_height, rs.image_width, sh, rs.sh_degree, campos, rs.prefiltered,
                                     rs.computer_pseudo_normal, **modes.forward_kw())
        else:
            ctx.views = None
            out = _debug_call(settings.debug, _C.rasterize_gaussians, _forward_args(settings, x), "snapshot_fw.dump",
                              "\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.",
                              _defer=defer, **modes.forward_kw())
            # one view: the backward takes the cameras from the settings (the same tensors); saving them (often views
            # of a larger buffer) would only add host time to every step
            x.update(dict.fromkeys(_CAMERAS))
        ctx.num_rendered = out[0]
        ctx.means2D = means2D if modes.absgrad else None      # the caller's tensor object: the backward sets .absgrad on it
        # cotangents of outputs the reference's backward ignores (num_contrib, normal, surface_xyz, weights, radii)
        # stay None instead of being materialised as zero tensors (5 fill kernels per step); the four image
        # cotangents are filled in by the backward when a loss does not touch one of them
        ctx.set_materialize_grads(False)
        ctx.out_shapes = tuple(t.shape for t in out[2:6])
        x.update(filter_3d=modes.filter_3d, radii=out[9], geomBuffer=out[10], binningBuffer=out[11], imgBuffer=out[12])
        ctx.save_for_backward(*(x[n] for n in _SAVED), *(out[3:5] if modes.surface_grads else ()))
        return out[:10] + (tuple(out[13:15]) if modes.depth_stats else ())

    @staticmethod
    def backward(ctx, g_num_rendered, g_num_contrib, g_color, g_opacity, g_depth, g_feature, g_normal, g_surface_xyz,
                 g_weights, g_radii, *g_stats):
        rs, modes = (ctx.settings if ctx.views is None else ctx.settings[0]), ctx.modes
        t = dict(zip(_SAVED, ctx.saved_tensors))
        if ctx.views is None:
            t.update(viewmatrix=rs.viewmatrix, projmatrix=rs.projmatrix, campos=rs.campos)
        need = dict(zip(_INPUTS, ctx.needs_input_grad))
        images = tuple(torch.zeros(shape, dtype=torch.float32, device=t["means3D"].device) if g is None else g
                       for g, shape in zip((g_color, g_opacity, g_depth, g_feature), ctx.out_shapes))
        ex = None
        if _EXCHANGE is not None and ctx.views is None:
            if rs.debug or t["sh"].numel() == 0:
                raise RuntimeError("a gradient exchange is installed (set_grad_exchange) but this backward cannot take "
                                   "part in it (debug mode or no `shs` input): every rank must run the same collectives")
            ex = _EXCHANGE
        # the full backward when a geometry input needs a gradient or a gradient exchange is installed, otherwise the
        # appearance-only backward for the appearance inputs that need one: frozen geometry (means2D included) thus
        # pays only for the gradients it uses
        geometry = _EXCHANGE is not None or any(need[n] for n in _GEOMETRY)
        kw = {} if geometry else {"geometry": False,
                                  "appearance": (need["features"], need["colors_precomp"], need["sh"])}
        kw.update(modes.backward_kw(t["opacities"], need["means2D"] and geometry, g_stats))
        if ex is not None:
            kw["_out"] = {"sh_factor": ex[0].factor}
        if any(need[n] for n in _CAMERAS):
            kw["cam_grads"] = True
        # (appearance-only: the surface outputs depend only on the geometry, their cotangents have nothing to reach)
        surface = geometry and modes.surface_grads and (g_normal is not None or g_surface_xyz is not None)
        if surface:
            kw["surface"] = ((g_normal, g_surface_xyz) + ctx.saved_tensors[len(_SAVED):] +
                             ((rs.cx, rs.cy) if ctx.views is None else ()))

        def library_backward(num_rendered, geom, binning, img):
            if ctx.views is not None:
                return _C.rasterize_views_backward(
                    ctx.views[0], t["means3D"], t["features"], t["colors_precomp"], t["scales"], t["rotations"],
                    rs.scale_modifier, t["cov3Ds_precomp"], t["viewmatrix"], t["projmatrix"], ctx.views[1], *images,
                    t["sh"], rs.sh_degree, t["campos"], geom, binning, img, rs.backward_geometry, **kw)
            return _debug_call(rs.debug, _C.rasterize_gaussians_backward,
                               (rs.bg, t["means3D"], t["features"], t["radii"], t["colors_precomp"], t["scales"],
                                t["rotations"], rs.scale_modifier, t["cov3Ds_precomp"], t["viewmatrix"],
                                t["projmatrix"], rs.tanfovx, rs.tanfovy, *images, t["sh"], rs.sh_degree, t["campos"],
                                geom, num_rendered, binning, img, rs.backward_geometry, rs.debug),
                               "snapshot_bw.dump", "\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n",
                               **kw)
        grads = library_backward(ctx.num_rendered, t["geomBuffer"], t["binningBuffer"], t["imgBuffer"])
        if isinstance(ctx.num_rendered, _C.DeferredCount):
            ctx.num_rendered.resolve()          # after the backward kernels are in flight
            if ctx.num_rendered.overflowed:     # rare: re-run the forward with the exact size, differentiate that
                warnings.warn(f"deferred rasterization overflowed its binning buffer ({int(ctx.num_rendered)} instances); "
                              "forward re-run inside backward (cotangents come from the truncated first attempt)")
                out = _C.rasterize_gaussians(*_forward_args(rs, t),
                                             _min_capacity=int(ctx.num_rendered) + 4096, **modes.forward_kw(rerun=True))
                if surface:                     # the adjoint of the re-run's own surface pass
                    kw["surface"] = (g_normal, g_surface_xyz, out[3], out[4], rs.cx, rs.cy)
                grads = library_backward(out[0], *out[10:13])
        g = dict(zip(_LIB_GRADS, grads[:9]))
        if ex is not None:                      # SH gradient: gather the views' factors, rebuild the mean locally
            exchange, campos_all = ex
            exchange.gather_factors()
            g["sh"] = exchange.rebuild_sh(t["means3D"], campos_all, rs.sh_degree)
        if kw.get("absgrad"):
            _set_absgrad(ctx.means2D, grads[-1])
            grads = grads[:-1]
        # camera gradients come in the cameras' shapes: None for those that do not need one (or when none was computed)
        g.update((n, c.reshape(t[n].shape) if need[n] else None) for n, c in zip(_CAMERAS, grads[9:]))
        return tuple(g.get(n) for n in _INPUTS) + (None,) * (len(ctx.needs_input_grad) - len(_INPUTS))


def _refuse_camera_grad_with_exchange(*cameras):
    """A gradient exchange renders one view per rank; camera gradients are not part of it."""
    if _EXCHANGE is not None and torch.is_grad_enabled() and any(
            isinstance(t, torch.Tensor) and t.requires_grad for t in cameras):
        raise RuntimeError("camera gradients (a viewmatrix, projmatrix or campos that requires grad) cannot be combined "
                           "with an installed gradient exchange (set_grad_exchange)")


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
    rs = raster_settings
    modes = _modes(means3D.shape[0], cov3Ds_precomp, rs.computer_pseudo_normal, surface_grads, antialiasing, filter_3d,
                   ray_depth, depth_stats, absgrad)
    _refuse_camera_grad_with_exchange(rs.viewmatrix, rs.projmatrix, rs.campos)
    inputs = (means3D, means2D, features, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
              rs.viewmatrix, rs.projmatrix, rs.campos)
    # decided here: inside the node's forward, grad mode is always off
    defer = (not rs.debug and _DEFER_COUNT and torch.is_grad_enabled()
             and any(isinstance(t, torch.Tensor) and t.requires_grad for t in inputs))
    return _Rasterize.apply(*inputs, raster_settings, modes, defer)


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
    `MAX_VIEWS` views or V·P >= 2^30 rows.  The modes are those of rasterize_gaussians and apply to every view (each
    view with its own depth planes); `means2D.absgrad` is then [V,P,2], and depth2 and median_depth [V,1,H,W]."""
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
    modes = _modes(means3D.shape[0], cov3D_precomp, settings[0].computer_pseudo_normal, surface_grads, antialiasing,
                   filter_3d, ray_depth, depth_stats, absgrad)
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
    if tuple(means2D.shape) != (V, P, 3):
        raise ValueError(f"rasterize_views: means2D must be [V,P,3] = {(V, P, 3)}, got {tuple(means2D.shape)}")
    for name, t in (("features", features), ("colors_precomp", colors_precomp)):
        if t.dim() == 3 and t.shape[0] != V:
            raise ValueError(f"rasterize_views: per-view {name} must have V = {V} rows, got {t.shape[0]}")
    # stacked here, outside the node, so that autograd routes each view's camera gradients to that view's tensors
    cameras = (torch.stack([s.viewmatrix for s in settings]), torch.stack([s.projmatrix for s in settings]),
               torch.stack([s.campos for s in settings]))
    return _Rasterize.apply(means3D, means2D, features, shs, colors_precomp, opacities, scales, rotations,
                            cov3D_precomp, *cameras, tuple(settings), modes, False)


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
