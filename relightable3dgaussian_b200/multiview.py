"""Multi-view consistency losses of PGSR (Chen et al., "PGSR: Planar-based Gaussian Splatting for Efficient and
High-Fidelity Surface Reconstruction", 2024), fused for sm_90a (csrc/multiview.cu).  Not part of the reference surface.

  consistency_loss(depth, normal, gray, settings, pairs, pixel_noise_threshold=1.0) -> (geo [B], photo [B])

For each (reference r, neighbour n) pair, every pixel of view r with depth D is reprojected into view n, its depth
D' sampled there and reprojected back: the geometric term is the weighted pixel error phi of that round trip, over
the pixels where it is below `pixel_noise_threshold`.  On those pixels, the plane through the pixel's point with the
pixel's normal gives a homography into view n; the photometric term is 1 - NCC of the 7x7 grey patch around the pixel
against its warp in the neighbour's grey image, over the pixels where it is below 0.9.  Each pixel is weighted by
exp(-phi) (no gradient) and each term is averaged over its valid pixels.  The exact definition is in
include/r3dg_b200.h (r3dg_multiview_*).  Gradients flow to `depth` (including the neighbour's depth at the four
bilinear taps of the reprojected pixel) and to `normal`; `gray` and the cameras get none.

One forward launch plus a fixed-order reduction on the device (no host read-back), and one backward launch that
recomputes the forward per pixel.  Under torch.use_deterministic_algorithms(True), read at call time, the backward
sums in fixed point and its gradients are bitwise reproducible.
"""
import ctypes
import numbers

import torch
from torch.autograd.function import once_differentiable

from . import _lib

MAX_PAIRS = 64          # R3DG_MAX_VIEWS (include/r3dg_b200.h)


def _host_pairs(pairs, V):
    """pairs as a list of B (r, n) int tuples with 0 <= r, n < V, checked on the host."""
    if isinstance(pairs, torch.Tensor):
        if pairs.is_cuda:
            raise ValueError("consistency_loss: pairs must be on the host (a sequence of (r, n) or a CPU tensor)")
        if pairs.dtype.is_floating_point or pairs.dtype.is_complex or pairs.dtype == torch.bool:
            raise TypeError(f"consistency_loss: pairs must be integers (got {pairs.dtype})")
        pairs = pairs.tolist()
    out = []
    for p in pairs:
        p = tuple(p)
        if len(p) != 2 or not all(isinstance(i, numbers.Integral) and not isinstance(i, bool) for i in p):
            raise TypeError(f"consistency_loss: each pair must be two ints (r, n), got {p!r}")
        out.append((int(p[0]), int(p[1])))
    if not 1 <= len(out) <= MAX_PAIRS:
        raise ValueError(f"consistency_loss: 1..{MAX_PAIRS} pairs per call (got {len(out)})")
    bad = [p for p in out if not (0 <= p[0] < V and 0 <= p[1] < V)]
    if bad:
        raise ValueError(f"consistency_loss: pairs {bad[:8]} index outside the {V} views")
    return out


def check_settings(fn, settings, V, H, W):
    """The V GaussianRasterizationSettings of V rendered H x W maps as a list, checked on the host (also used by
    tsdf.py)."""
    settings = list(settings)
    if len(settings) != V:
        raise ValueError(f"{fn}: {len(settings)} settings for {V} views")
    for v, s in enumerate(settings):
        if (s.image_height, s.image_width) != (H, W):
            raise ValueError(f"{fn}: settings[{v}] is {s.image_height}x{s.image_width}, the maps are {H}x{W}")
        if tuple(s.viewmatrix.shape) != (4, 4):
            raise ValueError(f"{fn}: settings[{v}].viewmatrix must be [4,4]")
        if not (s.tanfovx > 0 and s.tanfovy > 0):
            raise ValueError(f"{fn}: settings[{v}] has tanfovx / tanfovy <= 0")
    return settings


def view_matrices(settings, device):
    """The settings' row-vector view matrices as one float32 [V,16] tensor on `device`."""
    view = torch.stack([s.viewmatrix.detach().to(device=device, dtype=torch.float32) for s in settings])
    return view.reshape(len(settings), 16)


def _args(depth, normal, gray, view, cams, pairs, tau):
    V, _, H, W = depth.shape
    a = _lib.MultiviewArgs()
    a.V, a.H, a.W, a.B = V, H, W, len(pairs) // 2
    a.depth, a.normal, a.gray, a.viewmatrix = depth.data_ptr(), normal.data_ptr(), gray.data_ptr(), view.data_ptr()
    a.pair_cams, a.pairs = ctypes.addressof(cams), ctypes.addressof(pairs)
    a.pixel_noise_threshold = tau
    return a


class _Consistency(torch.autograd.Function):
    """(geo [B], photo [B], counts int32 [B,2]) from contiguous float32 depth [V,1,H,W], normal [V,3,H,W],
    gray [V,1,H,W] and view matrices [V,16]; `cams` and `pairs` are ctypes host arrays ([B][8] floats, [B][2] ints)."""

    @staticmethod
    def forward(ctx, depth, normal, gray, view, cams, pairs, tau):
        d, nrm, g, vm = (_lib.f32(t) for t in (depth, normal, gray, view))
        B, (V, _, H, W) = len(pairs) // 2, d.shape
        dev = d.device
        geo = torch.empty(B, dtype=torch.float32, device=dev)
        photo = torch.empty(B, dtype=torch.float32, device=dev)
        counts = torch.empty((B, 2), dtype=torch.int32, device=dev)
        work = _lib.scratch(_lib.load().r3dg_multiview_work_bytes(B, H, W), dev)
        a = _args(d, nrm, g, vm, cams, pairs, tau)
        a.geo, a.photo, a.counts, a.work, a.work_bytes = geo.data_ptr(), photo.data_ptr(), counts.data_ptr(), \
            work.data_ptr(), work.numel()
        _lib.call("r3dg_multiview_forward", dev, ctypes.byref(a), what="multiview consistency_loss")
        ctx.save_for_backward(d, nrm, g, vm, counts)
        ctx.cams, ctx.pairs, ctx.tau = cams, pairs, tau
        ctx.mark_non_differentiable(counts)
        return geo, photo, counts

    @staticmethod
    @once_differentiable
    def backward(ctx, dgeo, dphoto, _dcounts):
        d, nrm, g, vm, counts = ctx.saved_tensors
        V, _, H, W = d.shape
        dev = d.device
        B = len(ctx.pairs) // 2
        zero = torch.zeros(B, dtype=torch.float32, device=dev)
        dgeo = zero if dgeo is None else _lib.f32(dgeo)
        dphoto = zero if dphoto is None else _lib.f32(dphoto)
        dd = torch.empty_like(d)
        dn = torch.empty_like(nrm)
        a = _args(d, nrm, g, vm, ctx.cams, ctx.pairs, ctx.tau)
        a.counts, a.dL_dgeo, a.dL_dphoto = counts.data_ptr(), dgeo.data_ptr(), dphoto.data_ptr()
        a.dL_ddepth, a.dL_dnormal = dd.data_ptr(), dn.data_ptr()
        ws = None
        if torch.are_deterministic_algorithms_enabled():
            ws = _lib.scratch(_lib.load().r3dg_multiview_det_bytes(V, H, W), dev)
            a.deterministic, a.det_work, a.det_work_bytes = 1, ws.data_ptr(), ws.numel()
        _lib.call("r3dg_multiview_backward", dev, ctypes.byref(a), what="multiview consistency_loss backward")
        return (dd if ctx.needs_input_grad[0] else None, dn if ctx.needs_input_grad[1] else None,
                None, None, None, None, None)


def _prepare(depth, normal, gray, settings, pairs, pixel_noise_threshold):
    """Host-side checks (nothing touches the device) and the call's inputs."""
    fn = "consistency_loss"
    for name, t, C in (("depth", depth, 1), ("normal", normal, 3), ("gray", gray, 1)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{fn}: {name} must be a tensor")
        if t.dtype != torch.float32:
            raise TypeError(f"{fn}: {name} must be float32 (got {t.dtype})")
        if t.dim() != 4 or t.shape[1] != C:
            raise ValueError(f"{fn}: {name} must be [V,{C},H,W] (got {tuple(t.shape)})")
    V, _, H, W = depth.shape
    for name, t in (("normal", normal), ("gray", gray)):
        if (t.shape[0], t.shape[2], t.shape[3]) != (V, H, W):
            raise ValueError(f"{fn}: {name} {tuple(t.shape)} disagrees with depth {tuple(depth.shape)}")
    if V == 0 or H == 0 or W == 0:
        raise ValueError(f"{fn}: empty maps {tuple(depth.shape)}")
    settings = check_settings(fn, settings, V, H, W)
    tau = float(pixel_noise_threshold)
    if not tau >= 0.0:
        raise ValueError(f"{fn}: pixel_noise_threshold must be >= 0 (got {pixel_noise_threshold})")
    plist = _host_pairs(pairs, V)
    for name, t in (("depth", depth), ("normal", normal), ("gray", gray)):
        if not t.is_cuda:
            raise ValueError(f"{fn}: {name} must be a CUDA tensor")
        if t.device != depth.device:
            raise ValueError(f"{fn}: {name} is on {t.device}, depth on {depth.device}")
    cams = (ctypes.c_float * (8 * len(plist)))()
    idx = (ctypes.c_int * (2 * len(plist)))()
    for b, (r, n) in enumerate(plist):
        sr, sn = settings[r], settings[n]
        cams[8 * b: 8 * b + 8] = [sr.tanfovx, sr.tanfovy, sr.cx, sr.cy, sn.tanfovx, sn.tanfovy, sn.cx, sn.cy]
        idx[2 * b], idx[2 * b + 1] = r, n
    return view_matrices(settings, depth.device), cams, idx, tau


def consistency_loss(depth, normal, gray, settings, pairs, pixel_noise_threshold=1.0):
    """PGSR's multi-view geometric and photometric losses for B (reference, neighbour) pairs of V rendered views.

    depth [V,1,H,W]: camera z (e.g. out_depth / opacity in ray-depth mode, or the median depth);
    normal [V,3,H,W]: world-frame normals (normalised here, so the rasterizer's premultiplied normal feature works);
    gray [V,1,H,W]: ground-truth grey images (no gradient); all float32 CUDA tensors on one device.
    settings: the V GaussianRasterizationSettings the views were rendered with (viewmatrix, tanfovx, tanfovy, cx, cy
    and the image size are read; the cameras get no gradient).  pairs: B (r, n) view indices, 1 <= B <= 64; r = n and
    repeated views are allowed.  Returns (geo [B], photo [B]); apply the weights and reductions of your choice
    (PGSR: 0.03 * geo.mean() + 0.15 * photo.mean())."""
    view, cams, idx, tau = _prepare(depth, normal, gray, settings, pairs, pixel_noise_threshold)
    geo, photo, _ = _Consistency.apply(depth, normal, gray, view, cams, idx, tau)
    return geo, photo
