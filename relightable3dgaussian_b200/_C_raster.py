"""Drop-in replacement for the reference's pybind module `r3dg_rasterization._C`
(r3dg-rasterization/ext.cpp:15-19): same three function names, positional arguments and return
tuples as rasterize_points.cu:36-141 / :143-235 / :237-256, implemented on top of the C ABI of
libr3dg_b200.so (include/r3dg_b200.h) with torch used only for device memory and streams.

Differences that are not observable through the reference's Python wrapper
(gaussian_renderer/r3dg_rasterization.py):
  * the three returned byte buffers have our own opaque layout;
  * outputs are allocated uninitialised (every element is written by the kernels) instead of with
    torch::full / torch::zeros;
  * work is enqueued on torch's current stream (the reference uses the legacy default stream);
  * the binning buffer is sized speculatively from the previous call and the instance count is
    read back once, after everything has been enqueued — the pipeline itself never synchronises;
    a missed speculation re-runs the forward (synchronous path: immediately; deferred path: in the
    autograd backward, before differentiating).

Under torch.use_deterministic_algorithms(True), read at call time, both calls run the library's
deterministic mode: out_weights and the nine gradients are then bitwise reproducible (the reference's
float atomics make them run-to-run nondeterministic).  Its workspace comes from the torch allocator.

One view and V views of the same Gaussians (rasterize_views / rasterize_views_backward) run through the same two
host paths, _forward and _backward: the library treats a one-view call as V = 1.

The modes below are not part of the reference surface.  Each is off by default, so the reference's wrapper, which
passes none of them, gets the reference's calls (ray_depth: unless its process default is set).

`geometry=False` on the two backward functions runs the library's appearance-only backward: only the colour / feature /
SH gradients, for training with frozen geometry.  Nothing is allocated for the six geometry gradients, which come back
None, and of dL_dfeatures, dL_dcolors, dL_dsh only those `appearance` = (features, colors, sh) asks for are computed (the
others are None too); the opacity, depth and surface cotangents are not read.

`antialiasing=True` on all four functions multiplies each Gaussian's opacity by
rho = sqrt(max(det(cov2D) / det(cov2D + 0.3 I), 2.5e-5)), the opacity compensation of the fixed 0.3 px^2 dilation; the
backward must be called with the forward's flag.

`absgrad=True` on the two backward functions also computes the absolute screen-space gradients dL_dmeans2D_abs (AbsGS,
gsplat's absgrad): per Gaussian and view, the sum over pixels of |dL/dmean2D.x| and |dL/dmean2D.y|, [P,2] or [V,P,2],
returned as one more element after all others (None with geometry=False, which never computes it).

`filter_3d=` on all four functions runs the library's 3D smoothing filter
(Mip-Splatting): a [P] or [P,1] fp32 CUDA tensor of per-Gaussian filter sizes f, shared by every view (filter3d.py).
Each Gaussian is drawn with scales sqrt(s^2 + f^2) and its opacity times sqrt(prod_k s_k^2 / (s_k^2 + f^2)).  The
backward takes the forward's tensor again and, with it, the forward's `opacities`; f gets no gradient.

`ray_depth=True` on all four functions: each Gaussian adds, at each pixel, the camera z where it peaks along the pixel's
ray, tz + p . (pixel - mean2D) with the per-Gaussian depth plane p = conic (T0 Sigma w_z, T1 Sigma w_z), instead of its
centre's tz; out_depth, out_surface_xyz and out_normal change.  A forward's None (the default) takes the process default
(set_ray_depth, off unless set), so the reference's wrapper follows it; a backward's None takes the forward's mode from
the geometry buffer's size.

`depth_stats=True` on the two forward functions also renders, per pixel, depth2 = sum w d^2 over the composited entries
(d: the depth the call composites, tz or the ray-depth plane) and the median depth (d of the entry at which the
transmittance falls through 0.5), [1,H,W] or [V,1,H,W]; the two images follow every other element of the returned
tuple.  None and False are off, and there is no process default: the reference's wrapper, which unpacks a fixed tuple,
never sees them.  The backward functions take their cotangents as `dL_dout_depth2` and `dL_dout_median_depth` (None:
zeros; only the geometry half reads them) and `depth_stats=None` for the forward's setting, read from the image
buffer's size.
"""
import ctypes
import warnings

import torch

from . import _lib

_state = {}          # per-device instance-count statistics + pinned readback slots
_SLOTS = 64
_LEARN = 8           # forwards per (P, W, H) shape that always take the synchronous read-back (learn the counts)
_HEADROOM = 4.0      # deferred mode: binning capacity = _HEADROOM x the largest count seen for the shape


def _dev_state(device):
    key = device.index if device.index is not None else torch.cuda.current_device()
    st = _state.get(key)
    if st is None:
        st = {"capacity": 0, "pinned": torch.zeros(_SLOTS, dtype=torch.int32).pin_memory(), "next": 0,
              "shape": None, "seen": 0, "rmax": 0, "pending": None, "overflows": 0}
        _state[key] = st
    return st


def _observe(st, rendered, P):
    """Running statistics of the instance count for the current shape (sizes the next binning buffer)."""
    st["seen"] += 1
    st["rmax"] = max(st["rmax"], int(rendered))
    st["capacity"] = max(int(rendered * 1.25) + 4096, 4 * P + 4096)


class DeferredCount:
    """`num_rendered` of a forward whose read-back has not been waited for yet (opt-in, see
    rasterizer.set_deferred_count).  int() / resolve() waits for the forward's event.  The binning
    buffer of a deferred forward is sized _HEADROOM x the largest count any view of this shape has
    produced (HBM is plentiful on an 80 GB H100: 6 B per instance); should a view still overflow it, nothing
    out of bounds was written, `overflowed` is set and the autograd backward re-runs the forward
    with the exact size before differentiating (rasterizer._Rasterize.backward)."""

    def __init__(self, event, slot_view, capacity, state, P):
        self._event, self._slot, self._capacity, self._state, self._P = event, slot_view, capacity, state, P
        self._value = None
        self.overflowed = False

    def resolve(self):
        if self._value is None:
            self._event.synchronize()
            self._value = int(self._slot.item())
            _observe(self._state, self._value, self._P)
            if self._state.get("pending") is self:
                self._state["pending"] = None
            if self._value > self._capacity:
                self.overflowed = True
                self._state["overflows"] += 1
        return self._value

    __int__ = __index__ = resolve

    def __repr__(self):
        return f"DeferredCount({self._value if self._value is not None else 'pending'})"


def _check_filter_3d(filter_3d, P, cov3D_precomp):
    """`filter_3d` as the library takes it ([P] fp32, contiguous, on the GPU), or None when absent.  Raises ValueError,
    before anything is enqueued, for a wrong length (e.g. a filter computed before densification changed P), a CPU,
    non-fp32 or non-contiguous tensor, one that requires grad (no gradient flows to it), or together with
    cov3D_precomp (the filter is defined on scales)."""
    if filter_3d is None:
        return None
    if not isinstance(filter_3d, torch.Tensor):
        raise ValueError("filter_3d must be a tensor or None")
    if cov3D_precomp is not None and cov3D_precomp.numel() != 0:
        raise ValueError("filter_3d is defined on scales and cannot be combined with cov3D_precomp")
    if tuple(filter_3d.shape) not in ((P,), (P, 1)):
        raise ValueError(f"filter_3d must have shape [{P}] or [{P},1] (one value per Gaussian), got "
                         f"{list(filter_3d.shape)}: recompute it after the number of Gaussians changed")
    if not filter_3d.is_cuda or filter_3d.dtype != torch.float32 or not filter_3d.is_contiguous():
        raise ValueError(f"filter_3d must be a contiguous float32 CUDA tensor, got {filter_3d.dtype} on "
                         f"{filter_3d.device}{'' if filter_3d.is_contiguous() else ' (not contiguous)'}")
    if filter_3d.requires_grad:
        raise ValueError("filter_3d must not require grad: the rasterizer computes no gradient for it (detach it)")
    return filter_3d


def _prep(t, name):
    if t is None or t.numel() == 0:
        return t
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def _shared_args(a, views, cams, W, H, degree, scale_modifier, background, means3D, features, colors, scales,
                 rotations, cov3D_precomp, viewmatrix, projmatrix, sh, campos):
    """Preps the inputs the forward and the backward share and enters them, with the sizes and the first view's
    tan_fov*, into the argument struct `a` (RasterFwdArgs or RasterBwdArgs).  A one-view call (`views` False) leaves
    V = 0; a V-view call enters its camera table, each row {tan_fovx, tan_fovy, cx, cy}, and whether features / colors
    are per view ([V,P,*]).  Returns what the caller holds until the call is enqueued: the prepped inputs and the
    table."""
    features_pv = views and features.dim() == 3
    colors_pv = views and colors is not None and colors.numel() != 0 and colors.dim() == 3
    background = _prep(background, "background"); means3D = _prep(means3D, "means3D"); sh = _prep(sh, "sh")
    colors = _prep(colors, "colors"); features = _prep(features, "features"); scales = _prep(scales, "scales")
    rotations = _lib.aligned16(_prep(rotations, "rotations")); cov3D_precomp = _prep(cov3D_precomp, "cov3D_precomp")
    viewmatrix = _prep(viewmatrix, "viewmatrix"); projmatrix = _prep(projmatrix, "projmatrix")
    campos = _prep(campos, "campos")
    a.background = _lib.ptr(background); a.means3D = _lib.ptr(means3D); a.shs = _lib.ptr(sh)
    a.colors_precomp = _lib.ptr(colors); a.features = _lib.ptr(features); a.scales = _lib.ptr(scales)
    a.rotations = _lib.ptr(rotations); a.cov3D_precomp = _lib.ptr(cov3D_precomp)
    a.viewmatrix = _lib.ptr(viewmatrix); a.projmatrix = _lib.ptr(projmatrix); a.campos = _lib.ptr(campos)
    a.P, a.S, a.D, a.W, a.H = means3D.size(0), features.size(-1), int(degree), W, H
    a.M = sh.size(1) if sh.numel() != 0 else 0
    a.scale_modifier, a.tan_fovx, a.tan_fovy = float(scale_modifier), float(cams[0][0]), float(cams[0][1])
    keep = [background, means3D, sh, colors, features, scales, rotations, cov3D_precomp, viewmatrix, projmatrix, campos]
    if views:
        table = (ctypes.c_float * (4 * len(cams)))(*(float(x) for c in cams for x in c))   # [V][4]
        keep.append(table)
        a.V, a.view_cams = len(cams), ctypes.cast(table, ctypes.c_void_p)
        a.features_per_view, a.colors_per_view = int(features_pv), int(colors_pv)
    return keep


_RAY_DEPTH = False      # process default of the ray-depth mode (set_ray_depth)


def set_ray_depth(enabled):
    """Process default of the ray-depth mode for every forward that does not pass `ray_depth` (rasterizer.set_ray_depth
    sets it).  It reaches every caller of this module, the reference's own wrapper over dropin/r3dg_rasterization
    included; each backward takes the mode of its forward from the geometry buffer."""
    global _RAY_DEPTH
    _RAY_DEPTH = bool(enabled)


def ray_depth_default():
    return _RAY_DEPTH


def _fwd_ray_depth(ray_depth):
    """A forward's mode: its keyword, or the process default when it passes none (None)."""
    return _RAY_DEPTH if ray_depth is None else bool(ray_depth)


def _buffer_bytes(P, S, W, H, V, ray_depth=False, depth_stats=False, absgrad=False):
    """(geometry buffer, image buffer, backward deterministic workspace) bytes of a call over V views of P Gaussians
    with S feature channels at W x H, in these modes.  A mode's buffer is always larger than the default one of the same
    shape, which is how the two functions below tell a buffer's mode from its size."""
    lib = _lib.load()
    geom = (lib.r3dg_raster_ray_depth_geom_bytes if ray_depth else lib.r3dg_raster_views_geom_bytes)(P, S, V)
    img = (lib.r3dg_raster_depth_stats_img_bytes if depth_stats else lib.r3dg_raster_views_img_bytes)(W, H, V)
    det = (lib.r3dg_raster_ray_depth_bwd_det_bytes if ray_depth else lib.r3dg_raster_bwd_det_bytes)(V * P, S)
    if absgrad:                 # absgrad's fixed-point sums follow the gradient rows'
        det += lib.r3dg_raster_bwd_det_absgrad_bytes(V * P)
    return geom, img, det


def _geom_ray_depth(ray_depth, geomBuffer, P, S, W, H, V):
    """A backward's ray-depth mode: its keyword, or (None) that of the forward that made `geomBuffer`."""
    if ray_depth is not None:
        return bool(ray_depth)
    return geomBuffer.numel() >= _buffer_bytes(P, S, W, H, V, ray_depth=True)[0]


def _img_depth_stats(depth_stats, imageBuffer, P, S, W, H, V):
    """A backward's depth-statistics setting: its keyword, or (None) that of the forward that made `imageBuffer`."""
    if depth_stats is not None:
        return bool(depth_stats)
    return imageBuffer.numel() >= _buffer_bytes(P, S, W, H, V, depth_stats=True)[1]


def _forward(*, views, background, means3D, features, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
             viewmatrix, projmatrix, cams, H, W, sh, degree, campos, prefiltered, computer_pseudo_normal, debug,
             capacity, pinned, defer, antialiasing, filter_3d, ray_depth, depth_stats):
    """The forward of the len(cams) views `cams` = [(tan_fovx, tan_fovy, cx, cy), ...]: one view (`views` False,
    outputs in the one-view shapes) or V views (outputs with a leading V).  Sizes the binning buffer for `capacity`
    instances and re-runs with room to spare while the counts, read back into the pinned int32 `pinned` (one per
    view), exceed it.  Returns the 12 outputs after num_rendered (then the two depth-statistics images), the event
    recorded once the counts are copied, and the counts as a list: None when `defer`, which returns after the first
    attempt without waiting."""
    lib = _lib.load()
    V, P, S = len(cams), means3D.size(0), features.size(-1)
    filter_3d = _check_filter_3d(filter_3d, P, cov3D_precomp)
    ray_depth = _fwd_ray_depth(ray_depth)
    dev = means3D.device
    a = _lib.RasterFwdArgs()
    keep = _shared_args(a, views, cams, W, H, degree, scale_modifier, background, means3D, features, colors, scales,
                        rotations, cov3D_precomp, viewmatrix, projmatrix, sh, campos)
    opacity = _prep(opacity, "opacity")
    a.opacities = _lib.ptr(opacity)
    a.cx, a.cy = float(cams[0][2]), float(cams[0][3])
    a.prefiltered = int(bool(prefiltered)); a.computer_pseudo_normal = int(bool(computer_pseudo_normal))
    a.debug = int(bool(debug)); a.antialiasing = int(bool(antialiasing)); a.ray_depth = int(bool(ray_depth))
    a.filter_3d = _lib.ptr(filter_3d)

    lead = (V,) if views else ()
    f32 = dict(dtype=torch.float32, device=dev)
    out_color = torch.empty(lead + (3, H, W), **f32)
    out_opacity = torch.empty(lead + (1, H, W), **f32)
    out_depth = torch.empty(lead + (1, H, W), **f32)
    out_feature = torch.empty(lead + (S, H, W), **f32)
    out_normal = torch.empty(lead + (3, H, W), **f32)
    out_surface_xyz = torch.empty(lead + (3, H, W), **f32)
    out_weights = torch.empty(lead + (P, 1), **f32)
    radii = torch.empty(lead + (P,), dtype=torch.int32, device=dev)
    geom_bytes, img_bytes, _ = _buffer_bytes(P, S, W, H, V, ray_depth, depth_stats)
    geomBuffer = torch.empty((geom_bytes,), dtype=torch.uint8, device=dev)
    imgBuffer = torch.empty((img_bytes,), dtype=torch.uint8, device=dev)
    stats = ()
    if depth_stats:
        stats = (torch.empty(lead + (1, H, W), **f32), torch.empty(lead + (1, H, W), **f32))    # depth2, median depth
        a.depth_stats, a.out_depth2, a.out_median_depth = 1, stats[0].data_ptr(), stats[1].data_ptr()
    a.out_color = out_color.data_ptr(); a.out_opacity = out_opacity.data_ptr()
    a.out_depth = out_depth.data_ptr(); a.out_feature = _lib.ptr(out_feature)
    a.out_normal = out_normal.data_ptr(); a.out_surface_xyz = out_surface_xyz.data_ptr()
    a.out_weights = _lib.ptr(out_weights); a.radii = _lib.ptr(radii); a.n_contrib = None
    a.geom = geomBuffer.data_ptr(); a.geom_bytes = geomBuffer.numel()
    a.img = imgBuffer.data_ptr(); a.img_bytes = imgBuffer.numel()
    det_ws = _lib.det_workspace(a, lib.r3dg_raster_fwd_det_bytes(V * P), dev)
    a.num_rendered_host = pinned.data_ptr()
    stream = torch.cuda.current_stream(dev)
    while True:
        # this module's torch.empty, not _lib.scratch: tests substitute it to hand the forward a reused binning buffer
        binningBuffer = torch.empty((lib.r3dg_raster_binning_bytes(capacity),), dtype=torch.uint8, device=dev)
        a.binning = binningBuffer.data_ptr(); a.binning_bytes = binningBuffer.numel()
        # recorded by the library right after the last view's count is copied, a quarter into the forward
        ev = torch.cuda.Event()
        ev.record(stream)                 # (creates the underlying cudaEvent_t; re-recorded inside the call)
        a.count_ready_event = ev.cuda_event
        _lib.call("r3dg_raster_forward", dev, ctypes.byref(a),
                  what="rasterize_views" if views else "rasterize_gaussians")
        if defer:                         # opt-in: let the host run ahead; the caller resolves the count later
            counts = None
            break
        if debug:
            stream.synchronize()
        else:
            ev.synchronize()              # the one read-back: the counts are part of the return tuple.  The host
                                          # resumes while the compositor still runs and can enqueue the loss / backward
        counts = pinned.tolist()
        if sum(counts) <= capacity:
            break
        capacity = int(sum(counts) * 1.25) + 4096       # speculation missed: rerun with room to spare
    off = lib.r3dg_raster_views_img_n_contrib_offset(W, H, V)
    n_contrib = imgBuffer[off:off + 4 * V * H * W].view(torch.int32).view(lead + (H, W))   # view, like the reference
    return (n_contrib, out_color, out_opacity, out_depth, out_feature, out_normal, out_surface_xyz, out_weights, radii,
            geomBuffer, binningBuffer, imgBuffer) + stats, ev, counts


def rasterize_gaussians(background, means3D, features, colors, opacity, scales, rotations,
                        scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                        cx, cy, image_height, image_width, sh, degree, campos, prefiltered,
                        computer_pseudo_normal, debug, _defer=False, _min_capacity=None, *, antialiasing=False,
                        filter_3d=None, ray_depth=None, depth_stats=None):
    """== RasterizeGaussiansCUDA (rasterize_points.cu:36-141).  Returns the 13-tuple
    (rendered, n_contrib, out_color, out_opacity, out_depth, out_feature, out_normal,
     out_surface_xyz, out_weights, radii, geomBuffer, binningBuffer, imgBuffer), with depth_stats then depth2 [1,H,W]
    and median_depth [1,H,W].  The modes: see the module notes."""
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")   # rasterize_points.cu:62-64
    P = means3D.size(0)
    H, W = int(image_height), int(image_width)
    st = _dev_state(means3D.device)
    shape = (P, W, H)
    if st["shape"] != shape:             # new model size / resolution (e.g. after densification): re-learn the counts
        st.update(shape=shape, seen=0, rmax=0, capacity=0)
    prev = st["pending"]
    if prev is not None:                 # a deferred forward whose backward never ran: account for it now
        prev.resolve()
        if prev.overflowed:
            warnings.warn("a deferred-count forward overflowed its binning buffer and was never differentiated; "
                          "its images were truncated (use the synchronous path for forwards without backward)")
    if st["seen"] < _LEARN:
        _defer = False                   # learn the instance counts of this shape with the synchronous read-back first
    if _min_capacity is not None:
        capacity = int(_min_capacity)
    elif _defer:
        capacity = max(int(st["rmax"] * _HEADROOM) + 4096, 4 * P + 4096)
    else:
        capacity = max(st["capacity"], 4 * P + 4096)
    slot = st["next"]
    st["next"] = (slot + 1) % _SLOTS
    pinned = st["pinned"][slot:slot + 1]
    out, ev, counts = _forward(
        views=False, background=background, means3D=means3D, features=features, colors=colors, opacity=opacity,
        scales=scales, rotations=rotations, scale_modifier=scale_modifier, cov3D_precomp=cov3D_precomp,
        viewmatrix=viewmatrix, projmatrix=projmatrix, cams=[(tan_fovx, tan_fovy, cx, cy)], H=H, W=W, sh=sh,
        degree=degree, campos=campos, prefiltered=prefiltered, computer_pseudo_normal=computer_pseudo_normal,
        debug=debug, capacity=capacity, pinned=pinned, defer=_defer, antialiasing=antialiasing, filter_3d=filter_3d,
        ray_depth=ray_depth, depth_stats=depth_stats)
    if _defer:
        rendered = DeferredCount(ev, pinned, capacity, st, P)
        st["pending"] = rendered
    else:
        rendered = counts[0]
        _observe(st, rendered, P)
    return (rendered,) + out


def _backward(*, views, background, means3D, features, colors, scales, rotations, scale_modifier, cov3D_precomp,
              viewmatrix, projmatrix, cams, dL_dout_color, dL_dout_opacity, dL_dout_depth, dL_dout_feature, sh, degree,
              campos, geomBuffer, binningBuffer, imageBuffer, backward_geometry, debug, _out, cam_grads, surface,
              surface_work, principal, geometry, appearance, antialiasing, absgrad, filter_3d, opacities, ray_depth,
              depth_stats, dL_dout_depth2, dL_dout_median_depth):
    """The backward of a _forward over the len(cams) views `cams` (only each view's tan_fov* is read here; `principal`
    is the first view's (cx, cy), or None).  Returns the nine gradients of rasterize_views_backward (one view: in the
    one-view shapes), the V-view camera gradients (empty unless `cam_grads`) and (dL_dmeans2D_abs,) with absgrad, ()
    without.  `_out`, `surface` and `surface_work` are those of rasterize_gaussians_backward (`surface` without the
    principal point)."""
    if not geometry and (cam_grads or _out is not None):
        raise ValueError("the appearance-only backward (geometry=False) computes no camera gradient and takes no `_out`")
    lib = _lib.load()
    V, P, S = len(cams), means3D.size(0), features.size(-1)
    filter_3d = _check_filter_3d(filter_3d, P, cov3D_precomp)
    if filter_3d is not None and (opacities is None or opacities.numel() != P):
        raise ValueError("the backward with filter_3d needs the forward's opacities ([P] or [P,1])")
    H, W = dL_dout_color.size(-2), dL_dout_color.size(-1)
    ray_depth = _geom_ray_depth(ray_depth, geomBuffer, P, S, W, H, V)
    depth_stats = _img_depth_stats(depth_stats, imageBuffer, P, S, W, H, V)
    if not depth_stats and (dL_dout_depth2 is not None or dL_dout_median_depth is not None):
        raise ValueError("cotangents of depth2 / median_depth need a forward with depth_stats=True")
    dev = means3D.device
    a = _lib.RasterBwdArgs()
    keep = _shared_args(a, views, cams, W, H, degree, scale_modifier, background, means3D, features, colors, scales,
                        rotations, cov3D_precomp, viewmatrix, projmatrix, sh, campos)
    M = a.M
    dL_dout_color = _prep(dL_dout_color, "dL_dout_color")
    dL_dout_opacity = _prep(dL_dout_opacity, "dL_dout_opacity")
    dL_dout_depth = _prep(dL_dout_depth, "dL_dout_depth")
    dL_dout_feature = _prep(dL_dout_feature, "dL_dout_feature")
    f32 = dict(dtype=torch.float32, device=dev)

    def _alloc(name, shape):
        # `_out` (dist.GradBucket views) lets the multi-GPU path have the kernels write straight
        # into the flat all-reduce buffer; every element is written, so empty() is enough.
        if _out is not None and name in _out:
            t = _out[name]
            assert t.is_contiguous() and tuple(t.shape) == tuple(shape) and t.dtype == torch.float32
            return t
        return torch.empty(shape, **f32)

    if not geometry:                      # appearance-only: the requested appearance gradients, nothing else
        need_features, need_colors, need_sh = appearance
        dL_dmeans3D = dL_dmeans2D = dL_dopacity = dL_dcov3D = dL_dscales = dL_drotations = None
        dL_dfeatures = torch.empty((V, P, S) if a.features_per_view else (P, S), **f32) if need_features else None
        dL_dcolors = (torch.empty((V, P, 3) if a.colors_per_view else (P, 3), **f32)
                      if need_colors and a.colors_precomp else None)
        dL_dsh = torch.empty((P, M, 3), **f32) if need_sh and M > 0 else None
        sh_factor = torch.empty((V, P, 3), **f32) if dL_dsh is not None and V > 1 else None
    else:
        dL_dmeans3D = _alloc("means3D", (P, 3))
        dL_dmeans2D = _alloc("means2D", ((V,) if views else ()) + (P, 3))
        dL_dfeatures = _alloc("features", (V, P, S) if a.features_per_view else (P, S))
        dL_dcolors = _alloc("colors", (V, P, 3) if a.colors_per_view else (P, 3))
        dL_dopacity = _alloc("opacity", (P, 1))
        dL_dcov3D = _alloc("cov3D", (P, 6))
        # multi-GPU exchange (dist.FactoredGradExchange): `_out["sh_factor"]` [P,3] asks for the view's rank-1
        # factor of dL_dsh INSTEAD of the dense tensor (returned empty), see r3dg_sh_grad_from_factors
        sh_factor = _out.get("sh_factor") if _out is not None else None
        if sh_factor is not None:
            assert sh_factor.is_contiguous() and tuple(sh_factor.shape) == (P, 3) and sh_factor.dtype == torch.float32
            if M == 0:
                raise RuntimeError("the SH-gradient factor needs `sh` inputs (colors_precomp has no SH gradient)")
            dL_dsh = _alloc("sh", (P, M, 3)) if "sh" in _out else torch.empty((0,), **f32)     # both on request (tests)
        else:
            dL_dsh = _alloc("sh", (P, M, 3))
            if V > 1 and M > 0:               # the library rebuilds dL_dsh from the views' rank-1 factors
                sh_factor = torch.empty((V, P, 3), **f32)
        dL_dscales = _alloc("scales", (P, 3))
        dL_drotations = _alloc("rotations", (P, 4))
    dL_dmeans2D_abs = torch.empty(((V,) if views else ()) + (P, 2), **f32) if absgrad and geometry else None
    # zeroed: a call with P = 0 writes nothing, otherwise the library overwrites every element
    cam = tuple(torch.zeros(shape, **f32) for shape in ((V, 4, 4), (V, 4, 4), (V, 3))) if cam_grads else ()
    # (appearance-only with nothing to compute: no call, e.g. S = 0 features the only input that needs a gradient)
    if P != 0 and (geometry or any(_lib.ptr(t) for t in (dL_dfeatures, dL_dcolors, dL_dsh))):
        a.backward_geometry = int(bool(backward_geometry)); a.debug = int(bool(debug))
        a.antialiasing = int(bool(antialiasing)); a.ray_depth = int(bool(ray_depth))
        if filter_3d is not None:
            opacities = _prep(opacities, "opacities")
            a.filter_3d, a.opacities = _lib.ptr(filter_3d), _lib.ptr(opacities)
        a.dL_dout_color = _lib.ptr(dL_dout_color); a.dL_dout_opacity = _lib.ptr(dL_dout_opacity)
        a.dL_dout_depth = _lib.ptr(dL_dout_depth); a.dL_dout_feature = _lib.ptr(dL_dout_feature)
        a.dL_dmeans2D = _lib.ptr(dL_dmeans2D); a.dL_dcolors = _lib.ptr(dL_dcolors)
        a.dL_dopacity = _lib.ptr(dL_dopacity); a.dL_dmeans3D = _lib.ptr(dL_dmeans3D)
        a.dL_dfeatures = _lib.ptr(dL_dfeatures); a.dL_dcov3D = _lib.ptr(dL_dcov3D); a.dL_dsh = _lib.ptr(dL_dsh)
        a.dL_dscales = _lib.ptr(dL_dscales); a.dL_drotations = _lib.ptr(dL_drotations)
        a.dL_dsh_factor = _lib.ptr(sh_factor)
        a.geom = geomBuffer.data_ptr(); a.geom_bytes = geomBuffer.numel()
        a.img = imageBuffer.data_ptr(); a.img_bytes = imageBuffer.numel()
        a.binning = binningBuffer.data_ptr(); a.binning_bytes = binningBuffer.numel()
        a.dL_dmeans2D_abs = _lib.ptr(dL_dmeans2D_abs)
        if depth_stats and geometry:                    # (the appearance-only backward reads neither cotangent)
            like = dL_dout_depth
            dL_dout_depth2, dL_dout_median_depth = (torch.zeros_like(like) if g is None else _prep(g, name) for g, name in
                                                    ((dL_dout_depth2, "dL_dout_depth2"),
                                                     (dL_dout_median_depth, "dL_dout_median_depth")))
            a.depth_stats = 1
            a.dL_dout_depth2, a.dL_dout_median_depth = dL_dout_depth2.data_ptr(), dL_dout_median_depth.data_ptr()
        det_bytes = _buffer_bytes(P, S, W, H, V, ray_depth, depth_stats, dL_dmeans2D_abs is not None)[2]
        det_ws = _lib.det_workspace(a, det_bytes, dev)
        if cam:
            cam_ws = _lib.scratch(lib.r3dg_raster_cam_grad_bytes(P, V), dev)
            a.dL_dviewmatrix, a.dL_dprojmatrix, a.dL_dcampos = (t.data_ptr() for t in cam)
            a.cam_work, a.cam_work_bytes = cam_ws.data_ptr(), cam_ws.numel()
        surface_ws = _surface_args(a, surface if geometry else None, W, H, V, dev, surface_work, principal=principal)
        _lib.call("r3dg_raster_backward", dev, ctypes.byref(a),
                  what="rasterize_views_backward" if views else "rasterize_gaussians_backward")
    elif dL_dmeans2D_abs is not None:                   # P = 0: nothing to write
        dL_dmeans2D_abs.zero_()
    return (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dfeatures, dL_dcov3D, dL_dsh,
            dL_dscales, dL_drotations), cam, ((dL_dmeans2D_abs,) if absgrad else ())


def rasterize_gaussians_backward(background, means3D, features, radii, colors, scales, rotations,
                                 scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
                                 tan_fovy, dL_dout_color, dL_dout_opacity, dL_dout_depth,
                                 dL_dout_feature, sh, degree, campos, geomBuffer, R, binningBuffer,
                                 imageBuffer, backward_geometry, debug, _out=None, cam_grads=False, surface=None,
                                 surface_work=None, geometry=True, appearance=(True, True, True), *, antialiasing=False,
                                 absgrad=False, filter_3d=None, opacities=None, ray_depth=None, depth_stats=None,
                                 dL_dout_depth2=None, dL_dout_median_depth=None):
    """== RasterizeGaussiansBackwardCUDA (rasterize_points.cu:143-235).  Returns the 9-tuple
    (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dfeatures, dL_dcov3D, dL_dsh,
     dL_dscales, dL_drotations).  With `cam_grads=True` (not part of the reference surface) three camera gradients
    follow: dL_dviewmatrix [4,4], dL_dprojmatrix [4,4] and dL_dcampos [3], in the element order of `viewmatrix`,
    `projmatrix` and `campos`.  `surface` (not part of the reference surface either) differentiates the pseudo-normal
    and surface-xyz outputs: (dL_dout_normal, dL_dout_surface_xyz, out_opacity, out_depth, cx, cy) with the forward's
    opacity and depth images; a cotangent may be None.  `surface_work` optionally supplies the workspace
    (r3dg_raster_surface_grad_bytes), e.g. to read the combined depth and opacity cotangents afterwards.  With absgrad,
    dL_dmeans2D_abs [P,2] is the last element.  The modes, and the forward's `opacities` the filter needs: see the
    module notes."""
    grads, cam, extra = _backward(
        views=False, background=background, means3D=means3D, features=features, colors=colors, scales=scales,
        rotations=rotations, scale_modifier=scale_modifier, cov3D_precomp=cov3D_precomp, viewmatrix=viewmatrix,
        projmatrix=projmatrix, cams=[(tan_fovx, tan_fovy)], dL_dout_color=dL_dout_color,
        dL_dout_opacity=dL_dout_opacity, dL_dout_depth=dL_dout_depth, dL_dout_feature=dL_dout_feature, sh=sh,
        degree=degree, campos=campos, geomBuffer=geomBuffer, binningBuffer=binningBuffer, imageBuffer=imageBuffer,
        backward_geometry=backward_geometry, debug=debug, _out=_out, cam_grads=cam_grads,
        surface=surface and surface[:4], surface_work=surface_work,
        principal=surface[4:6] if surface is not None and len(surface) == 6 else None, geometry=geometry,
        appearance=appearance, antialiasing=antialiasing, absgrad=absgrad, filter_3d=filter_3d, opacities=opacities,
        ray_depth=ray_depth, depth_stats=depth_stats, dL_dout_depth2=dL_dout_depth2,
        dL_dout_median_depth=dL_dout_median_depth)
    return grads + tuple(t[0] for t in cam) + extra


def _surface_args(a, surface, W, H, V, device, work=None, principal=None):
    """Enters the pseudo-normal / surface-xyz cotangents `surface` = (dL_dout_normal, dL_dout_surface_xyz, opacity,
    depth) (or none) and their workspace into the backward arguments `a`; returns the cotangents and the workspace,
    which the caller holds until the call is enqueued.  Both cotangents None: nothing is entered.  `principal` = (cx, cy)
    is the principal point of a one-view call (V = 1), which the library reads from `a.cx, a.cy`, and is required
    then: a V-view call (V > 1) reads every view's own from its camera table."""
    if surface is None or (surface[0] is None and surface[1] is None):
        return None
    if V <= 1 and principal is None:
        raise ValueError("the surface gradients of a one-view call need the forward's principal point (cx, cy)")
    g_normal, g_xyz = (None if g is None else _prep(g, name) for g, name in
                       ((surface[0], "dL_dout_normal"), (surface[1], "dL_dout_surface_xyz")))
    opacity, depth = _prep(surface[2], "out_opacity"), _prep(surface[3], "out_depth")
    if work is None:
        work = _lib.scratch(_lib.load().r3dg_raster_surface_grad_bytes(W, H, V), device)
    a.dL_dout_normal, a.dL_dout_surface_xyz = _lib.ptr(g_normal), _lib.ptr(g_xyz)
    a.fwd_opacity, a.fwd_depth = _lib.ptr(opacity), _lib.ptr(depth)
    if principal is not None:
        a.cx, a.cy = float(principal[0]), float(principal[1])
    a.surface_work, a.surface_work_bytes = work.data_ptr(), work.numel()
    return g_normal, g_xyz, opacity, depth, work


def mark_visible(means3D, viewmatrix, projmatrix):
    """== markVisible (rasterize_points.cu:237-256): bool[P] = view-space z > 0.2."""
    P = means3D.size(0)
    present = torch.zeros((P,), dtype=torch.bool, device=means3D.device)
    if P != 0:
        means3D = _prep(means3D, "means3D"); viewmatrix = _prep(viewmatrix, "viewmatrix")
        projmatrix = _prep(projmatrix, "projmatrix")
        _lib.call("r3dg_mark_visible", means3D.device, P, means3D.data_ptr(), viewmatrix.data_ptr(),
                  projmatrix.data_ptr(), present.data_ptr(), what="mark_visible")
    return present


def debug_intermediate(name, P, S, W, H, geomBuffer, imgBuffer, binningBuffer, num_rendered=0):
    """Parity introspection (r3dg_raster_debug_copy): returns a dense tensor of one named
    intermediate in the reference's element layout."""
    lib = _lib.load()
    T = ((W + 15) // 16) * ((H + 15) // 16)
    spec = {"depths": (0, torch.float32, (P,)), "clamped": (1, torch.uint8, (P, 3)),
            "means2D": (3, torch.float32, (P, 2)), "conic_opacity": (5, torch.float32, (P, 4)),
            "rgb": (6, torch.float32, (P, 3)), "tiles_touched": (7, torch.int32, (P,)),
            "point_offsets": (8, torch.int32, (P,)), "point_list": (9, torch.int32, (num_rendered,)),
            "point_list_keys": (10, torch.int64, (num_rendered,)),
            "final_T": (13, torch.float32, (H, W)), "n_contrib": (14, torch.int32, (H, W)),
            "ranges": (15, torch.int32, (T, 2)), "bwd_work": (16, torch.int32, (T, 2)),
            "bwd_order": (17, torch.int32, (2 * T,)), "bmask": (18, torch.uint8, (num_rendered,)),
            "cmask": (19, torch.uint8, (num_rendered,)), "brects": (20, torch.int32, (P, 2)),
            "composited": (22, torch.uint8, (P,)), "median_pos": (23, torch.int32, (H, W))}[name]
    if name == "median_pos" and not _img_depth_stats(None, imgBuffer, P, S, W, H, 1):
        raise RuntimeError("debug_intermediate(median_pos) needs the image buffer of a forward with depth_stats=True")
    out = torch.empty(spec[2], dtype=spec[1], device=geomBuffer.device)
    if out.numel() == 0:
        return out
    nbytes = out.numel() * out.element_size()
    stream = torch.cuda.current_stream(geomBuffer.device)
    # a ray-depth geometry buffer has the mode's layout (records and gradient rows one float4 wider)
    copy = lib.r3dg_raster_ray_depth_debug_copy if _geom_ray_depth(None, geomBuffer, P, S, W, H, 1) else lib.r3dg_raster_debug_copy
    with torch.cuda.device(geomBuffer.device):
        rc = copy(spec[0], P, S, W, H, geomBuffer.data_ptr(), imgBuffer.data_ptr(),
                                        binningBuffer.data_ptr(), binningBuffer.numel(), out.data_ptr(),
                                        nbytes, stream.cuda_stream)
    if rc < 0:
        raise RuntimeError(f"debug_intermediate({name}) failed: {rc}")
    return out


# ---- several views of the same Gaussians in one call (r3dg_raster_forward / _backward with V > 1) ----------------------
_views_capacity = {}     # (device, P, W, H, V) -> binning capacity that held the last call of that shape


def rasterize_views(background, means3D, features, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                    viewmatrix, projmatrix, cams, image_height, image_width, sh, degree, campos, prefiltered,
                    computer_pseudo_normal, _min_capacity=None, *, antialiasing=False, filter_3d=None, ray_depth=None,
                    depth_stats=None):
    """V views of one set of Gaussians in one forward.  background [V,3], viewmatrix / projmatrix [V,4,4], campos [V,3],
    cams: V tuples (tan_fovx, tan_fovy, cx, cy); features [P,S] or [V,P,S], colors [P,3] or [V,P,3] (or empty).
    Returns (num_rendered: list of V ints, n_contrib [V,H,W], out_color [V,3,H,W], out_opacity [V,1,H,W],
    out_depth [V,1,H,W], out_feature [V,S,H,W], out_normal [V,3,H,W], out_surface_xyz [V,3,H,W], out_weights [V,P,1],
    radii [V,P], geomBuffer, binningBuffer, imgBuffer), with depth_stats then depth2 [V,1,H,W] and median_depth
    [V,1,H,W].  Always synchronous: the V counts are read back once.  The modes apply to every view."""
    V, P = len(cams), means3D.size(0)
    H, W = int(image_height), int(image_width)
    dev = means3D.device
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), P, W, H, V)
    capacity = int(_min_capacity) if _min_capacity is not None else max(_views_capacity.get(key, 0), 4 * V * P + 4096)
    pinned = torch.zeros((V,), dtype=torch.int32).pin_memory()
    out, _, rendered = _forward(
        views=True, background=background, means3D=means3D, features=features, colors=colors, opacity=opacity,
        scales=scales, rotations=rotations, scale_modifier=scale_modifier, cov3D_precomp=cov3D_precomp,
        viewmatrix=viewmatrix, projmatrix=projmatrix, cams=cams, H=H, W=W, sh=sh, degree=degree, campos=campos,
        prefiltered=prefiltered, computer_pseudo_normal=computer_pseudo_normal, debug=False, capacity=capacity,
        pinned=pinned, defer=False, antialiasing=antialiasing, filter_3d=filter_3d, ray_depth=ray_depth,
        depth_stats=depth_stats)
    _views_capacity[key] = max(int(sum(rendered) * 1.25) + 4096, 4 * V * P + 4096)
    return (rendered,) + out


def rasterize_views_backward(background, means3D, features, colors, scales, rotations, scale_modifier, cov3D_precomp,
                             viewmatrix, projmatrix, cams, dL_dout_color, dL_dout_opacity, dL_dout_depth,
                             dL_dout_feature, sh, degree, campos, geomBuffer, binningBuffer, imageBuffer,
                             backward_geometry, cam_grads=False, surface=None, surface_work=None, geometry=True,
                             appearance=(True, True, True), *, antialiasing=False, absgrad=False, filter_3d=None,
                             opacities=None, ray_depth=None, depth_stats=None, dL_dout_depth2=None,
                             dL_dout_median_depth=None):
    """Backward of rasterize_views.  Returns (dL_dmeans2D [V,P,3], dL_dcolors, dL_dopacity [P,1], dL_dmeans3D,
    dL_dfeatures, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations): dL_dfeatures / dL_dcolors have the shape of their
    input ([P,*] summed over the views, or [V,P,*] per view); every other leaf gradient is the fp32 sum over the views
    in view order; dL_dsh is rebuilt from the views' rank-1 factors.  With `cam_grads=True` each view's camera
    gradients follow, never summed: dL_dviewmatrix [V,4,4], dL_dprojmatrix [V,4,4], dL_dcampos [V,3].  `surface` =
    (dL_dout_normal, dL_dout_surface_xyz, out_opacity, out_depth), all [V,*,H,W] (a cotangent may be None), and
    `surface_work` are those of rasterize_gaussians_backward; each view uses its own principal point from `cams` (with
    one view, cams[0]'s, entered as the call's cx, cy).  With absgrad, dL_dmeans2D_abs [V,P,2] is the last element.
    The modes: see the module notes."""
    grads, cam, extra = _backward(
        views=True, background=background, means3D=means3D, features=features, colors=colors, scales=scales,
        rotations=rotations, scale_modifier=scale_modifier, cov3D_precomp=cov3D_precomp, viewmatrix=viewmatrix,
        projmatrix=projmatrix, cams=cams, dL_dout_color=dL_dout_color, dL_dout_opacity=dL_dout_opacity,
        dL_dout_depth=dL_dout_depth, dL_dout_feature=dL_dout_feature, sh=sh, degree=degree, campos=campos,
        geomBuffer=geomBuffer, binningBuffer=binningBuffer, imageBuffer=imageBuffer,
        backward_geometry=backward_geometry, debug=False, _out=None, cam_grads=cam_grads, surface=surface,
        surface_work=surface_work, principal=cams[0][2:4], geometry=geometry, appearance=appearance,
        antialiasing=antialiasing, absgrad=absgrad, filter_3d=filter_3d, opacities=opacities, ray_depth=ray_depth,
        depth_stats=depth_stats, dL_dout_depth2=dL_dout_depth2, dL_dout_median_depth=dL_dout_median_depth)
    return grads + cam + extra
