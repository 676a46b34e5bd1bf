"""G-buffer-guided a-trous denoising of per-pixel shading (include/r3dg_b200.h, DENOISE; DESIGN.md §4.32).

Per-pixel shading at a few samples per pixel (shading.shade_pixels, lights.shade_pixels) carries independent noise at
every pixel.  `atrous` is a cross-bilateral a-trous wavelet filter (Dammertz et al. 2010, the spatial filter of SVGF)
whose edge-stopping weights come from the normal, point, mask and optional feature guides only, never from the noisy
signal: it is linear in the image, and its gradient is the exact transposed filter, computed by a gather on the GPU
(no atomics, bitwise reproducible).  `denoise_shading` denoises the demodulated terms of a shading call and recomposes
pbr = base_color / pi * diffuse_light + specular, so the albedo texture is never blurred.

Everything runs in the library's sm_90a kernels; there is no CPU path.  Inputs are checked before anything is
launched."""
import ctypes
import math

import torch

from . import _lib

MAX_VIEWS = 64           # R3DG_MAX_VIEWS
MAX_CHANNELS = 8         # R3DG_DENOISE_MAX_CHANNELS
MAX_FEATURES = 8         # R3DG_DENOISE_MAX_FEATURES
MAX_PASSES = 6           # R3DG_DENOISE_MAX_PASSES


def _planar(t, name, lead=None, channels=None):
    """The shape check of a planar image [C,H,W] or [V,C,H,W]: (leading shape, H, W) and C."""
    if not isinstance(t, torch.Tensor) or t.dim() not in (3, 4):
        raise ValueError(f"{name} must be a [C,H,W] or [V,C,H,W] tensor, got {getattr(t, 'shape', type(t))}")
    shape = (tuple(t.shape[:-3]), t.shape[-2], t.shape[-1])
    if lead is not None and shape != lead:
        raise ValueError(f"{name} {tuple(t.shape)} does not match the image's views and size {lead}")
    if channels is not None and t.shape[-3] != channels:
        raise ValueError(f"{name} must have {channels} channels, got {tuple(t.shape)}")
    return shape, t.shape[-3]


def _sigma(v, name):
    v = float(v)
    if not (math.isfinite(v) and v > 0):
        raise ValueError(f"{name} must be finite and > 0 (got {v})")
    return v


def _dev(t):
    """`t` as contiguous float32 [V,C,H,W], detached."""
    x = _lib.f32(t)
    return x if x.dim() == 4 else x.unsqueeze(0)


def _prepare(x, normal, points, mask, features, passes, sigma_normal, sigma_plane, sigma_features):
    """Every check of an atrous call, before anything is launched; the call's DenoiseArgs without its pointers."""
    lead, C = _planar(x, "x")
    if not 1 <= C <= MAX_CHANNELS:
        raise ValueError(f"x must have 1 to {MAX_CHANNELS} channels, got {C}")
    V = x.shape[0] if x.dim() == 4 else 1
    if not 1 <= V <= MAX_VIEWS:
        raise ValueError(f"atrous takes 1 to {MAX_VIEWS} views per call (got {V})")
    _planar(normal, "normal", lead, 3)
    _planar(points, "points", lead, 3)
    F = 0
    if features is not None:
        _, F = _planar(features, "features", lead)
        if F > MAX_FEATURES:
            raise ValueError(f"features must have 0 to {MAX_FEATURES} channels, got {F}")
    if mask is not None and (mask.dtype not in (torch.bool, torch.uint8) or tuple(mask.shape) != lead[0] + lead[1:]):
        raise ValueError(f"mask must be bool or uint8 {lead[0] + lead[1:]}, got {mask.dtype} {tuple(mask.shape)}")
    if isinstance(passes, bool) or int(passes) != passes or not 1 <= passes <= MAX_PASSES:
        raise ValueError(f"passes must be an integer in 1..{MAX_PASSES} (got {passes})")
    sn, sx, sf = (_sigma(v, n) for v, n in ((sigma_normal, "sigma_normal"), (sigma_plane, "sigma_plane"),
                                             (sigma_features, "sigma_features")))
    H, W = lead[1], lead[2]
    if V * H * W * max(C, F) >= 2 ** 31:
        raise ValueError(f"V H W max(C, F) = {V * H * W * max(C, F)} must stay below 2^31 (32-bit indices)")
    given = [t for t in (x, normal, points, mask, features) if t is not None]
    if not all(t.is_cuda for t in given):
        raise RuntimeError("atrous needs CUDA tensors (the denoiser runs on the GPU only)")
    if len({t.device for t in given}) != 1:
        raise ValueError(f"atrous's tensors are on different devices: {sorted({str(t.device) for t in given})}")
    a = _lib.DenoiseArgs()
    a.V, a.H, a.W, a.C, a.F, a.L = V, H, W, C, F, int(passes)
    a.sigma_normal, a.sigma_plane, a.sigma_features = sn, sx, sf
    return a


class _Atrous(torch.autograd.Function):
    """One node for the L passes: gradient to x only (the guides are detached)."""

    @staticmethod
    def forward(ctx, x, a, normal, points, mask, features):
        dev = x.device
        xs, n, p = _dev(x), _dev(normal), _dev(points)
        f = None if features is None or a.F == 0 else _dev(features)
        m = None
        if mask is not None:
            m = mask.detach().contiguous()
            m = m.view(torch.uint8) if m.dtype == torch.bool else m
        y = torch.empty_like(xs)
        work = _lib.scratch(_lib.load().r3dg_denoise_work_bytes(a.V, a.H, a.W, a.C, a.F, a.L), dev)
        a.normal, a.points, a.mask, a.features = n.data_ptr(), p.data_ptr(), _lib.ptr(m), _lib.ptr(f)
        a.x, a.y, a.work, a.work_bytes = xs.data_ptr(), y.data_ptr(), work.data_ptr(), work.numel()
        _lib.call("r3dg_denoise_forward", dev, ctypes.byref(a), what="atrous")
        ctx.save_for_backward(work)
        ctx.args, ctx.shape = (a.V, a.H, a.W, a.C, a.F, a.L, a.sigma_normal, a.sigma_plane, a.sigma_features), x.shape
        return y.reshape(x.shape)

    @staticmethod
    def backward(ctx, g):
        (work,) = ctx.saved_tensors
        a = _lib.DenoiseArgs()
        a.V, a.H, a.W, a.C, a.F, a.L, a.sigma_normal, a.sigma_plane, a.sigma_features = ctx.args
        gy = _lib.f32(g)
        dx = torch.empty_like(gy)
        a.dL_dy, a.dL_dx, a.work, a.work_bytes = gy.data_ptr(), dx.data_ptr(), work.data_ptr(), work.numel()
        _lib.call("r3dg_denoise_backward", gy.device, ctypes.byref(a), what="atrous backward")
        return dx.reshape(ctx.shape), None, None, None, None, None


def atrous(x, normal, points, mask=None, features=None, passes=4, sigma_normal=128.0, sigma_plane=0.1,
           sigma_features=0.1):
    """The G-buffer-guided a-trous filter of x [C,H,W] or [V,C,H,W] (1 <= C <= 8, 1 <= V <= 64).

    Guides of the same views and size: normal [..,3,H,W] (un-premultiplied, any length), points [..,3,H,W] (world-space
    surface points), mask [..,H,W] (bool or uint8; the mask shade_pixels takes) and features [..,F,H,W] (F <= 8, e.g.
    roughness).  `passes` passes of a 5 x 5 B-spline stencil at steps 1, 2, 4, ..., each tap weighted by
    max(n_p . n_q, 0)^sigma_normal (unit normals), exp(-t / sigma_plane) with t the sine of the tap's angle out of p's
    tangent plane, and exp(-|f_p - f_q|^2 / sigma_features^2), then normalised.  Masked pixels output 0 and their
    values of x are never read.  Returns y with x's shape; the gradient goes to x only, and is the exact transposed
    filter.  Everything is checked before anything is launched."""
    a = _prepare(x, normal, points, mask, features, passes, sigma_normal, sigma_plane, sigma_features)
    return _apply(x, a, normal, points, mask, features)


def _apply(x, a, normal, points, mask, features):
    return _Atrous.apply(x, a, normal.detach(), points.detach(), mask, None if features is None else features.detach())


def denoise_shading(out, base_color, roughness, normal, points, mask=None, passes=4, sigma_normal=128.0, sigma_plane=0.1,
                    sigma_features=0.1):
    """Denoise the output of shading.shade_pixels or lights.shade_pixels (or the sum of several such dicts).

    pbr = base_color / pi * diffuse_light + specular, so the filter runs on the demodulated terms: diffuse_light with
    the normal and point guides, specular with roughness [..,1,H,W] as a feature guide too, and pbr is recomposed from
    the undenoised base_color.  passes and the sigmas: as in `atrous`.  Returns dict(pbr, diffuse_light, specular).
    Gradients flow to base_color and, through the two denoised terms, into the shading call's backward."""
    opts = (passes, sigma_normal, sigma_plane, sigma_features)
    lead, _ = _planar(out["diffuse_light"], "diffuse_light")
    _planar(out["specular"], "specular", lead, 3)
    _planar(base_color, "base_color", lead, 3)
    _planar(roughness, "roughness", lead, 1)
    a_diffuse = _prepare(out["diffuse_light"], normal, points, mask, None, *opts)
    a_specular = _prepare(out["specular"], normal, points, mask, roughness, *opts)
    if not base_color.is_cuda or base_color.device != out["diffuse_light"].device:
        raise RuntimeError("base_color must be a CUDA tensor on the shading outputs' device")
    diffuse = _apply(out["diffuse_light"], a_diffuse, normal, points, mask, None)
    specular = _apply(out["specular"], a_specular, normal, points, mask, roughness)
    return {"pbr": base_color / math.pi * diffuse + specular, "diffuse_light": diffuse, "specular": specular}
