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
"""
import ctypes

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
    with the exact size before differentiating (rasterizer._RasterizeGaussians.backward)."""

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


def _ptr(t):
    """Device pointer of an optional tensor; empty tensors mean "absent" (NULL), like the
    reference (forward.cu:206,242)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def _det_workspace(nbytes, dev):
    """Workspace of the deterministic mode when torch.are_deterministic_algorithms_enabled(), else None."""
    if not torch.are_deterministic_algorithms_enabled():
        return None
    return torch.empty((nbytes,), dtype=torch.uint8, device=dev)


def _set_det(a, ws):
    if ws is not None:
        a.deterministic, a.det_work, a.det_work_bytes = 1, ws.data_ptr(), ws.numel()


def _prep(t, name):
    if t is None or t.numel() == 0:
        return t
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def rasterize_gaussians(background, means3D, features, colors, opacity, scales, rotations,
                        scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                        cx, cy, image_height, image_width, sh, degree, campos, prefiltered,
                        computer_pseudo_normal, debug, _defer=False, _min_capacity=None):
    """== RasterizeGaussiansCUDA (rasterize_points.cu:36-141).  Returns the 13-tuple
    (rendered, n_contrib, out_color, out_opacity, out_depth, out_feature, out_normal,
     out_surface_xyz, out_weights, radii, geomBuffer, binningBuffer, imgBuffer)."""
    lib = _lib.load()
    if means3D.ndimension() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")   # rasterize_points.cu:62-64
    P = means3D.size(0)
    S = features.size(1)
    H, W = int(image_height), int(image_width)
    dev = means3D.device
    means3D = _prep(means3D, "means3D")
    features = _prep(features, "features"); colors = _prep(colors, "colors")
    opacity = _prep(opacity, "opacity"); scales = _prep(scales, "scales")
    rotations = _prep(rotations, "rotations"); cov3D_precomp = _prep(cov3D_precomp, "cov3D_precomp")
    sh = _prep(sh, "sh"); background = _prep(background, "background")
    viewmatrix = _prep(viewmatrix, "viewmatrix"); projmatrix = _prep(projmatrix, "projmatrix")
    campos = _prep(campos, "campos")
    M = sh.size(1) if sh.numel() != 0 else 0

    f32 = dict(dtype=torch.float32, device=dev)
    out_color = torch.empty((3, H, W), **f32)
    out_opacity = torch.empty((1, H, W), **f32)
    out_depth = torch.empty((1, H, W), **f32)
    out_feature = torch.empty((S, H, W), **f32)
    out_normal = torch.empty((3, H, W), **f32)
    out_surface_xyz = torch.empty((3, H, W), **f32)
    out_weights = torch.empty((P, 1), **f32)
    radii = torch.empty((P,), dtype=torch.int32, device=dev)
    geomBuffer = torch.empty((lib.r3dg_raster_geom_bytes(P, S),), dtype=torch.uint8, device=dev)
    imgBuffer = torch.empty((lib.r3dg_raster_img_bytes(W, H),), dtype=torch.uint8, device=dev)

    st = _dev_state(dev)
    shape = (P, W, H)
    if st["shape"] != shape:             # new model size / resolution (e.g. after densification): re-learn the counts
        st.update(shape=shape, seen=0, rmax=0, capacity=0)
    prev = st["pending"]
    if prev is not None:                 # a deferred forward whose backward never ran: account for it now
        prev.resolve()
        if prev.overflowed:
            import warnings
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
    stream = torch.cuda.current_stream(dev)
    det_ws = _det_workspace(lib.r3dg_raster_fwd_det_bytes(P), dev)
    slot = st["next"]
    st["next"] = (slot + 1) % _SLOTS
    pinned = st["pinned"][slot:slot + 1]
    with torch.cuda.device(dev):
        while True:
            binningBuffer = torch.empty((lib.r3dg_raster_binning_bytes(capacity),), dtype=torch.uint8,
                                        device=dev)
            a = _lib.RasterFwdArgs()
            a.P, a.S, a.D, a.M, a.W, a.H = P, S, int(degree), M, W, H
            a.background = _ptr(background); a.means3D = _ptr(means3D); a.shs = _ptr(sh)
            a.colors_precomp = _ptr(colors); a.features = _ptr(features); a.opacities = _ptr(opacity)
            a.scales = _ptr(scales); a.rotations = _ptr(rotations); a.cov3D_precomp = _ptr(cov3D_precomp)
            a.viewmatrix = _ptr(viewmatrix); a.projmatrix = _ptr(projmatrix); a.campos = _ptr(campos)
            a.scale_modifier = float(scale_modifier); a.tan_fovx = float(tan_fovx)
            a.tan_fovy = float(tan_fovy); a.cx = float(cx); a.cy = float(cy)
            a.prefiltered = int(bool(prefiltered)); a.computer_pseudo_normal = int(bool(computer_pseudo_normal))
            a.debug = int(bool(debug))
            a.out_color = out_color.data_ptr(); a.out_opacity = out_opacity.data_ptr()
            a.out_depth = out_depth.data_ptr(); a.out_feature = _ptr(out_feature)
            a.out_normal = out_normal.data_ptr(); a.out_surface_xyz = out_surface_xyz.data_ptr()
            a.out_weights = _ptr(out_weights); a.radii = _ptr(radii); a.n_contrib = None
            a.geom = geomBuffer.data_ptr(); a.geom_bytes = geomBuffer.numel()
            a.img = imgBuffer.data_ptr(); a.img_bytes = imgBuffer.numel()
            a.binning = binningBuffer.data_ptr(); a.binning_bytes = binningBuffer.numel()
            a.num_rendered_host = pinned.data_ptr()
            # recorded by the library right after the count's D2H copy — a quarter into the forward, not at its end
            ev = torch.cuda.Event()
            ev.record(stream)             # (creates the underlying cudaEvent_t; re-recorded inside the call)
            a.count_ready_event = ev.cuda_event
            _set_det(a, det_ws)
            _lib.check(lib.r3dg_raster_forward(ctypes.byref(a), stream.cuda_stream), "rasterize_gaussians")
            if _defer:                    # opt-in: let the host run ahead; the count is resolved later
                rendered = DeferredCount(ev, pinned, capacity, st, P)
                st["pending"] = rendered
                break
            if debug:
                stream.synchronize()
            else:
                ev.synchronize()          # the one readback: num_rendered is part of the return tuple.  The host resumes
                                          # while the compositor still runs and can enqueue the loss / backward behind it
            rendered = int(pinned.item())
            if rendered <= capacity:
                break
            capacity = int(rendered * 1.25) + 4096      # speculation missed: rerun with room to spare
    if not _defer:
        _observe(st, rendered, P)
    off = lib.r3dg_raster_img_n_contrib_offset(W, H)
    n_contrib = imgBuffer[off:off + 4 * H * W].view(torch.int32).view(H, W)   # view, like the reference
    return (rendered, n_contrib, out_color, out_opacity, out_depth, out_feature, out_normal,
            out_surface_xyz, out_weights, radii, geomBuffer, binningBuffer, imgBuffer)


def rasterize_gaussians_backward(background, means3D, features, radii, colors, scales, rotations,
                                 scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
                                 tan_fovy, dL_dout_color, dL_dout_opacity, dL_dout_depth,
                                 dL_dout_feature, sh, degree, campos, geomBuffer, R, binningBuffer,
                                 imageBuffer, backward_geometry, debug, _out=None):
    """== RasterizeGaussiansBackwardCUDA (rasterize_points.cu:143-235).  Returns the 9-tuple
    (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dfeatures, dL_dcov3D, dL_dsh,
     dL_dscales, dL_drotations)."""
    lib = _lib.load()
    P = means3D.size(0)
    S = features.size(1)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    dev = means3D.device
    means3D = _prep(means3D, "means3D"); features = _prep(features, "features")
    colors = _prep(colors, "colors"); scales = _prep(scales, "scales")
    rotations = _prep(rotations, "rotations"); cov3D_precomp = _prep(cov3D_precomp, "cov3D_precomp")
    sh = _prep(sh, "sh"); background = _prep(background, "background")
    viewmatrix = _prep(viewmatrix, "viewmatrix"); projmatrix = _prep(projmatrix, "projmatrix")
    campos = _prep(campos, "campos")
    dL_dout_color = _prep(dL_dout_color, "dL_dout_color")
    dL_dout_opacity = _prep(dL_dout_opacity, "dL_dout_opacity")
    dL_dout_depth = _prep(dL_dout_depth, "dL_dout_depth")
    dL_dout_feature = _prep(dL_dout_feature, "dL_dout_feature")
    M = sh.size(1) if sh.numel() != 0 else 0

    f32 = dict(dtype=torch.float32, device=dev)

    def _alloc(name, shape):
        # `_out` (dist.GradBucket views) lets the multi-GPU path have the kernels write straight
        # into the flat all-reduce buffer; every element is written, so empty() is enough.
        if _out is not None and name in _out:
            t = _out[name]
            assert t.is_contiguous() and tuple(t.shape) == tuple(shape) and t.dtype == torch.float32
            return t
        return torch.empty(shape, **f32)

    dL_dmeans3D = _alloc("means3D", (P, 3))
    dL_dmeans2D = _alloc("means2D", (P, 3))
    dL_dfeatures = _alloc("features", (P, S))
    dL_dcolors = _alloc("colors", (P, 3))
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
    dL_dscales = _alloc("scales", (P, 3))
    dL_drotations = _alloc("rotations", (P, 4))
    if P != 0:
        a = _lib.RasterBwdArgs()
        a.P, a.S, a.D, a.M, a.W, a.H = P, S, int(degree), M, W, H
        a.background = _ptr(background); a.means3D = _ptr(means3D); a.shs = _ptr(sh)
        a.colors_precomp = _ptr(colors); a.features = _ptr(features); a.scales = _ptr(scales)
        a.rotations = _ptr(rotations); a.cov3D_precomp = _ptr(cov3D_precomp)
        a.viewmatrix = _ptr(viewmatrix); a.projmatrix = _ptr(projmatrix); a.campos = _ptr(campos)
        a.scale_modifier = float(scale_modifier); a.tan_fovx = float(tan_fovx); a.tan_fovy = float(tan_fovy)
        a.backward_geometry = int(bool(backward_geometry)); a.debug = int(bool(debug))
        a.dL_dout_color = _ptr(dL_dout_color); a.dL_dout_opacity = _ptr(dL_dout_opacity)
        a.dL_dout_depth = _ptr(dL_dout_depth); a.dL_dout_feature = _ptr(dL_dout_feature)
        a.dL_dmeans2D = _ptr(dL_dmeans2D); a.dL_dcolors = _ptr(dL_dcolors)
        a.dL_dopacity = _ptr(dL_dopacity); a.dL_dmeans3D = _ptr(dL_dmeans3D)
        a.dL_dfeatures = _ptr(dL_dfeatures); a.dL_dcov3D = _ptr(dL_dcov3D); a.dL_dsh = _ptr(dL_dsh)
        a.dL_dscales = _ptr(dL_dscales); a.dL_drotations = _ptr(dL_drotations)
        a.dL_dsh_factor = _ptr(sh_factor)
        a.geom = geomBuffer.data_ptr(); a.geom_bytes = geomBuffer.numel()
        a.img = imageBuffer.data_ptr(); a.img_bytes = imageBuffer.numel()
        a.binning = binningBuffer.data_ptr(); a.binning_bytes = binningBuffer.numel()
        det_ws = _det_workspace(lib.r3dg_raster_bwd_det_bytes(P, S), dev)
        _set_det(a, det_ws)
        stream = torch.cuda.current_stream(dev)
        with torch.cuda.device(dev):
            _lib.check(lib.r3dg_raster_backward(ctypes.byref(a), stream.cuda_stream),
                       "rasterize_gaussians_backward")
    return (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dfeatures, dL_dcov3D, dL_dsh,
            dL_dscales, dL_drotations)


def mark_visible(means3D, viewmatrix, projmatrix):
    """== markVisible (rasterize_points.cu:237-256): bool[P] = view-space z > 0.2."""
    lib = _lib.load()
    P = means3D.size(0)
    present = torch.zeros((P,), dtype=torch.bool, device=means3D.device)
    if P != 0:
        means3D = _prep(means3D, "means3D"); viewmatrix = _prep(viewmatrix, "viewmatrix")
        projmatrix = _prep(projmatrix, "projmatrix")
        stream = torch.cuda.current_stream(means3D.device)
        with torch.cuda.device(means3D.device):
            _lib.check(lib.r3dg_mark_visible(P, means3D.data_ptr(), viewmatrix.data_ptr(),
                                             projmatrix.data_ptr(), present.data_ptr(),
                                             stream.cuda_stream), "mark_visible")
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
            "cmask": (19, torch.uint8, (num_rendered,)), "brects": (20, torch.int32, (P, 2))}[name]
    out = torch.empty(spec[2], dtype=spec[1], device=geomBuffer.device)
    if out.numel() == 0:
        return out
    nbytes = out.numel() * out.element_size()
    stream = torch.cuda.current_stream(geomBuffer.device)
    with torch.cuda.device(geomBuffer.device):
        rc = lib.r3dg_raster_debug_copy(spec[0], P, S, W, H, geomBuffer.data_ptr(), imgBuffer.data_ptr(),
                                        binningBuffer.data_ptr(), binningBuffer.numel(), out.data_ptr(),
                                        nbytes, stream.cuda_stream)
    if rc < 0:
        raise RuntimeError(f"debug_intermediate({name}) failed: {rc}")
    return out
