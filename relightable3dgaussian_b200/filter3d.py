"""Mip-Splatting's 3D smoothing filter (Yu et al., "Mip-Splatting: Alias-free 3D Gaussian Splatting", CVPR 2024).

Nothing stops the optimiser from making a Gaussian much smaller than the finest pixel footprint any training camera
gave it; zoomed in, or rendered at a higher resolution, such Gaussians show up as speckle and erosion.  The 3D filter
dilates each Gaussian's covariance by f^2 I, f from the highest sampling rate at which a training camera saw it, and
scales its opacity so that the Gaussian keeps its integrated weight.

  compute_3d_filter(means3D, cameras) -> f [P,1]   the filter sizes, one CUDA pass over all (Gaussian, camera) pairs
                                                    (r3dg_filter3d_compute), with no host synchronisation;
  rasterize_gaussians(..., filter_3d=f)             the rasterizer draws the filtered Gaussians (rasterizer.py);
  fold(scales, opacities, f) -> (s', o')            the filtered scales and opacities in plain fp32 torch, the same
                                                    operations in the same order as the rasterizer, for consumers that
                                                    take no filter (visibility bake, PLY export, evaluation without the
                                                    training cameras).  A model folded this way renders bit for bit as
                                                    the filtered one.

The filter is a buffer, not a parameter: recompute it when the Gaussians or the cameras change (after densification,
after MCMC relocation, and every ~100 iterations after densification stops, as Mip-Splatting does).
"""
import ctypes

import numpy as np
import torch

from . import _lib


def _intrinsics(cam):
    """(fx, fy, cx, cy) of a training camera as its get_intrinsics() holds them (fp32), computed on the host from the
    camera's own attributes: fx, fy, cx, cy when it has them, otherwise a FoV camera's W / (2 tan(FoVx / 2)),
    H / (2 tan(FoVy / 2)) and (W / 2, H / 2).  A camera with neither is read through get_intrinsics()."""
    W, H = cam.image_width, cam.image_height
    fx = getattr(cam, "fx", None)
    if fx is not None:
        vals = (fx, cam.fy, cam.cx, cam.cy)
    elif hasattr(cam, "FoVx") and hasattr(cam, "FoVy"):
        vals = (W / (2 * np.tan(cam.FoVx * 0.5)), H / (2 * np.tan(cam.FoVy * 0.5)), W / 2, H / 2)
    else:
        K = cam.get_intrinsics().detach().cpu()
        vals = (K[0, 0], K[1, 1], K[0, 2], K[1, 2])
    return tuple(float(np.float32(float(v))) for v in vals)


def compute_3d_filter(means3D, cameras):
    """Mip-Splatting's compute_3D_filter on the GPU: f [P,1] (fp32, on means3D's device) for the Gaussians at
    `means3D` [P,3] and the training `cameras` (objects with `world_view_transform`, `image_width`, `image_height`
    and the intrinsics of get_intrinsics(), see _intrinsics).

    A (Gaussian, camera) pair is valid when the Gaussian's view-space depth z, formed exactly as the rasterizer forms
    its near-cull depth, is > 0.2 and its pixel position lies within 15 % of the image on every side.  d is the least z
    of the valid pairs (Gaussians no camera sees take the largest d of the others), and f = d / F * sqrt(0.2) with F the
    largest fx of all cameras.  Unlike Mip-Splatting, the pixel position uses each camera's own principal point
    (cx, cy), not (W/2, H/2); the two agree for FoV cameras.  Also unlike it, d is not capped at 1e5, and when no
    camera sees any Gaussian f is 0 everywhere (the unfiltered model) instead of an error.

    The host work is one torch.stack of the view matrices on the device and one copy of the [V,6] intrinsics table
    to it; nothing is read back, so the call does not wait for the GPU.  Two launches (none for P = 0); the result is
    bitwise reproducible, so every rank of a data-parallel run computes the same filter without a collective."""
    cameras = list(cameras)
    if not cameras:
        raise ValueError("compute_3d_filter needs at least one training camera")
    if means3D.dim() != 2 or means3D.shape[1] != 3:
        raise ValueError(f"means3D must be [P,3], got {list(means3D.shape)}")
    if not means3D.is_cuda:
        raise ValueError("means3D must be a CUDA tensor")
    dev = means3D.device
    means = _lib.f32(means3D)
    P, V = means.shape[0], len(cameras)
    out = torch.empty((P, 1), dtype=torch.float32, device=dev)
    if P == 0:
        return out
    views = torch.stack([c.world_view_transform.detach().to(device=dev, dtype=torch.float32) for c in cameras])
    views = views.reshape(V, 16).contiguous()
    rows = [_intrinsics(c) + (float(c.image_width), float(c.image_height)) for c in cameras]
    F = max(r[0] for r in rows)
    if not (F > 0 and np.isfinite(F)):
        raise ValueError(f"the largest focal length of the cameras must be finite and positive, got {F}")
    # pinned + non_blocking: the copy is enqueued on the stream without a host wait; the caching host allocator keeps
    # the pinned block alive until the copy has run
    table = torch.tensor(rows, dtype=torch.float32).pin_memory().to(dev, non_blocking=True)
    lib = _lib.load()
    tmp = _lib.scratch(lib.r3dg_filter3d_tmp_bytes(P), dev)
    _lib.call("r3dg_filter3d_compute", dev, P, V, means.data_ptr(), views.data_ptr(), table.data_ptr(),
              ctypes.c_float(F), out.data_ptr(), tmp.data_ptr(), tmp.numel(), what="compute_3d_filter")
    return out


def fold(scales, opacities, filter_3d):
    """(s', o'): the Gaussians the rasterizer draws with `filter_3d`, as plain fp32 torch operations in the
    rasterizer's order: q = s * s, g = f * f, e = q + g, s' = sqrt(e), r = q / e (1 where e = 0),
    coef = sqrt((r_0 r_1) r_2), o' = o * coef.  `scales` [P,3] and `opacities` [P,1] or [P] are the activated values
    (get_scaling, get_opacity), `filter_3d` [P,1] or [P].  Rendering (s', o') without a filter gives the same bits as
    rendering (s, o) with it.  f = 0 returns |s| and o.  The result is differentiable with respect to scales and
    opacities (except where s' = 0), not to the filter."""
    f = filter_3d.reshape(-1, 1)
    q = scales * scales
    e = q + f * f
    s_f = torch.sqrt(e)
    r = torch.where(e == 0, torch.ones_like(q), q / e)
    coef = torch.sqrt((r[:, 0] * r[:, 1]) * r[:, 2])
    return s_f, opacities * coef.reshape(opacities.shape)
