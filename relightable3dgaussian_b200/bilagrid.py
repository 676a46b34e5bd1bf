"""Bilateral-grid colour correction (Wang et al., "Bilateral Guided Radiance Field Processing", SIGGRAPH 2024), as
gsplat trains it with `--use_bilateral_grid`.

Real captures differ from image to image in exposure, white balance and tone curve.  Without a per-image correction
the optimiser explains those differences with the scene: floaters and view-dependent colour in stage 1, and base
colour, roughness and environment light in stage 2.  A bilateral grid per training image absorbs them in a small,
learnable, locally affine colour transform, used during training only and discarded for novel-view and relit renders.

  slice(grids, rgb, image_ids)   the corrected images, with gradients to rgb and to the grids (csrc/bilagrid.cu,
                                 r3dg_bilagrid_forward / _backward): one kernel forward, one or two backward,
                                 bitwise reproducible, no host synchronisation;
  BilateralGrid(num_images)      the identity-initialised grids as a Module, with forward() = slice and tv_loss().

Semantics (include/r3dg_b200.h): for pixel (px, py) of an image with colour (r, g, b), the 3x4 affine matrix A is the
trilinear interpolation of the image's grid at ((px + 0.5) / W, (py + 0.5) / H, 0.299 r + 0.587 g + 0.114 b) with
F.grid_sample's align_corners=True, padding_mode="border" mapping, and out = A (r, g, b, 1).
"""
import numbers

import torch
from torch.autograd.function import once_differentiable

from . import _lib

IDENTITY = (1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0)


def _host_ids(image_ids, n, G):
    """image_ids (an int, a sequence of ints or a CPU integer tensor) as a list of n ints in [0, G), checked on the
    host: nothing here touches the GPU."""
    if isinstance(image_ids, torch.Tensor):
        if image_ids.is_cuda:
            raise ValueError("slice: image_ids must be on the CPU (a Python int, a sequence or a CPU tensor), so that "
                             "their range is checked without waiting for the GPU")
        if image_ids.dtype.is_floating_point or image_ids.dtype.is_complex or image_ids.dtype == torch.bool:
            raise TypeError(f"slice: image_ids must be integers (got {image_ids.dtype})")
        ids = image_ids.reshape(-1).tolist()
    elif isinstance(image_ids, numbers.Integral) and not isinstance(image_ids, bool):
        ids = [int(image_ids)]
    else:
        ids = list(image_ids)
        if not all(isinstance(i, numbers.Integral) and not isinstance(i, bool) for i in ids):
            raise TypeError("slice: image_ids must be integers")
        ids = [int(i) for i in ids]
    if len(ids) != n:
        raise ValueError(f"slice: {len(ids)} image ids for {n} images")
    bad = [i for i in ids if not 0 <= i < G]
    if bad:
        raise ValueError(f"slice: image ids {bad[:8]} out of range [0, {G})")
    return ids


class _Slice(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids, rgb, ids):
        g, x = _lib.f32(grids), _lib.f32(rgb)
        G, _, L, GY, GX = g.shape
        N, _, H, W = x.shape
        out = torch.empty_like(x)
        _lib.call("r3dg_bilagrid_forward", x.device, G, N, H, W, GX, GY, L, g.data_ptr(), ids.data_ptr(), x.data_ptr(),
                  out.data_ptr(), what="bilagrid slice")
        ctx.save_for_backward(g, x, ids)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        g, x, ids = ctx.saved_tensors
        G, _, L, GY, GX = g.shape
        N, _, H, W = x.shape
        d = _lib.f32(dout)
        dgrids = torch.empty_like(g) if ctx.needs_input_grad[0] else None
        drgb = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        tmp = None            # the per-tile partial sub-grids of dL/dgrids
        if dgrids is not None:
            tmp = _lib.scratch(_lib.load().r3dg_bilagrid_tmp_bytes(G, N, H, W, GX, GY, L), x.device)
        _lib.call("r3dg_bilagrid_backward", x.device, G, N, H, W, GX, GY, L, g.data_ptr(), ids.data_ptr(), x.data_ptr(),
                  d.data_ptr(), _lib.ptr(drgb), _lib.ptr(dgrids), _lib.ptr(tmp), 0 if tmp is None else tmp.numel(),
                  what="bilagrid slice backward")
        return dgrids, drgb, None


def slice(grids, rgb, image_ids):
    """Apply each image's bilateral grid: grids [G,12,L,GY,GX] (gsplat's BilateralGrid.grids), rgb [N,3,H,W] or
    [3,H,W] (N = 1), both float32 CUDA tensors on one device (rgb may be non-contiguous), and image_ids: N indices in
    [0, G) as a Python int, a sequence of ints or a CPU integer tensor.  Returns the corrected images in rgb's shape.
    Gradients flow to rgb and to the grids, each only when autograd asks for it; repeated ids sum their gradients."""
    for name, t in (("grids", grids), ("rgb", rgb)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"slice: {name} must be a tensor")
        if t.dtype != torch.float32:
            raise TypeError(f"slice: {name} must be float32 (got {t.dtype})")
    if grids.dim() != 5 or grids.shape[1] != 12:
        raise ValueError(f"slice: grids must be [G,12,L,GY,GX] (got {tuple(grids.shape)})")
    if rgb.dim() not in (3, 4) or rgb.shape[-3] != 3:
        raise ValueError(f"slice: rgb must be [3,H,W] or [N,3,H,W] (got {tuple(rgb.shape)})")
    x = rgb if rgb.dim() == 4 else rgb.unsqueeze(0)
    ids = _host_ids(image_ids, x.shape[0], grids.shape[0])
    for name, t in (("grids", grids), ("rgb", rgb)):
        if not t.is_cuda:
            raise ValueError(f"slice: {name} must be a CUDA tensor")
    if grids.device != rgb.device:
        raise ValueError(f"slice: grids and rgb are on different devices ({grids.device}, {rgb.device})")
    # pinned + non_blocking: the copy is enqueued without a host wait; the caching host allocator keeps the pinned
    # block alive until it has run
    ids = torch.tensor(ids, dtype=torch.int32).pin_memory().to(rgb.device, non_blocking=True)
    out = _Slice.apply(grids, x, ids)
    return out if rgb.dim() == 4 else out.squeeze(0)


class BilateralGrid(torch.nn.Module):
    """One bilateral grid per training image (gsplat's BilateralGrid): `grids` [num_images, 12, grid_W, grid_Y, grid_X],
    initialised to the identity transform, so that an untrained grid returns its input bit for bit."""

    def __init__(self, num_images, grid_X=16, grid_Y=16, grid_W=8):
        super().__init__()
        ident = torch.tensor(IDENTITY, dtype=torch.float32).reshape(1, 12, 1, 1, 1)
        self.grids = torch.nn.Parameter(ident.repeat(num_images, 1, grid_W, grid_Y, grid_X))

    def forward(self, rgb, image_ids):
        """slice(self.grids, rgb, image_ids)."""
        return slice(self.grids, rgb, image_ids)

    def tv_loss(self):
        """Total variation of the grids: the sum over the luma, y and x axes of the mean squared forward difference.
        Plain torch: the grids are small (G x 24,576 floats at the defaults)."""
        return sum(torch.diff(self.grids, dim=d).square().mean() for d in (2, 3, 4))
