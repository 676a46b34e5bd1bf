"""Fused image-space loss terms of the reference's training loss (utils/loss_utils.py), with the reference's
signatures and return shapes, backed by sm_90a kernels:

  ssim(img1, img2, window_size=11, size_average=True)  (:32-63)  r3dg_ssim_forward / _backward (csrc/ssim.cu)
  first_order_edge_aware_loss(data, img)                (:104-105) r3dg_edge_aware_forward / _backward (csrc/smooth.cu)
  tv_loss(x)                                            (:113-117) r3dg_tv_forward / _backward (csrc/smooth.cu)

The reference calls ssim every training step (gaussian_renderer/render.py:150; twice in
gaussian_renderer/neilf.py:227,234) and as an evaluation metric (eval_nvs.py:72,
eval_relighting_syn4.py:191,195), and the two regularisers in stage 1 (render.py:170) and stage 2
(neilf.py:284,291,299,306,312).  Its callers import the names with `from utils.loss_utils import ...`, so
`install()` rebinds them in utils.loss_utils and in every module that already holds a copy (a 2-line plug-in, see
INTEGRATION.md).

Differences from the reference, all deliberate: results are computed in IEEE fp32 (cuDNN runs the reference's
convolutions in TF32 under torch's defaults), the reductions are deterministic, ssim(x, x) is exactly 1, and the
regularisers give exactly 0 (and zero gradients) on constant data.  Only what the call sites use is supported;
anything else raises instead of falling back to PyTorch.
"""
import sys

import torch
from torch.autograd.function import once_differentiable

from . import _lib

DEFAULT_MODULES = ("utils.loss_utils", "gaussian_renderer.render", "gaussian_renderer.neilf")
_saved = []            # (module, name, previous value) of every rebinding made by install()


def _check_cuda_f32(fn, name, t):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError(f"{fn}: {name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        raise TypeError(f"{fn}: {name} must be float32 (got {t.dtype})")


class _SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2, size_average):
        x, y = _lib.f32(img1), _lib.f32(img2)
        N = 1 if x.dim() == 3 else x.shape[0]
        C, H, W = x.shape[-3:]
        dev = x.device
        out = torch.empty(() if size_average else (N,), dtype=torch.float32, device=dev)
        tmp = _lib.scratch(max(_lib.load().r3dg_ssim_tmp_bytes(N, C, H, W), 1), dev)
        _lib.call("r3dg_ssim_forward", dev, N, C, H, W, x.data_ptr(), y.data_ptr(), int(size_average), out.data_ptr(),
                  tmp.data_ptr(), tmp.numel(), what="ssim")
        ctx.save_for_backward(x, y)
        ctx.size_average = size_average
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, y = ctx.saved_tensors
        N = 1 if x.dim() == 3 else x.shape[0]
        C, H, W = x.shape[-3:]
        g = _lib.f32(g)
        grads = []
        for need, a, b in ((ctx.needs_input_grad[0], x, y), (ctx.needs_input_grad[1], y, x)):   # dL/dimg2: img1 <-> img2
            d = None
            if need:
                d = torch.empty_like(a)
                _lib.call("r3dg_ssim_backward", x.device, N, C, H, W, a.data_ptr(), b.data_ptr(), int(ctx.size_average),
                          g.data_ptr(), d.data_ptr(), what="ssim backward")
            grads.append(d)
        return grads[0], grads[1], None


def ssim(img1, img2, window_size=11, size_average=True):
    """Drop-in for utils/loss_utils.py:32: mean SSIM of two [C,H,W] or [N,C,H,W] float32 CUDA images (0-dim), or
    per image ([N]) when size_average is False on 4-D input.  Gradients flow to both inputs."""
    if window_size != 11:
        raise ValueError(f"ssim: only window_size=11 is supported (got {window_size})")
    for name, t in (("img1", img1), ("img2", img2)):
        _check_cuda_f32("ssim", name, t)
        if t.dim() not in (3, 4):
            raise ValueError(f"ssim: {name} must be [C,H,W] or [N,C,H,W] (got {tuple(t.shape)})")
    if img1.shape != img2.shape:
        raise ValueError(f"ssim: shapes differ: {tuple(img1.shape)} vs {tuple(img2.shape)}")
    if img1.device != img2.device:
        raise ValueError(f"ssim: inputs are on different devices ({img1.device}, {img2.device})")
    if not size_average and img1.dim() == 3:
        # the reference's ssim_map.mean(1).mean(1).mean(1) has no third dimension to reduce here either
        raise ValueError("ssim: size_average=False needs [N,C,H,W] input")
    return _SSIM.apply(img1, img2, bool(size_average))


class _EdgeAware(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, img):
        d, i = _lib.f32(data), _lib.f32(img)
        (Cd, H, W), Ci = d.shape, i.shape[0]
        dev = d.device
        out = torch.empty((), dtype=torch.float32, device=dev)
        tmp = _lib.scratch(max(_lib.load().r3dg_edge_aware_tmp_bytes(Cd, Ci, H, W), 1), dev)
        _lib.call("r3dg_edge_aware_forward", dev, Cd, Ci, H, W, d.data_ptr(), i.data_ptr(), out.data_ptr(),
                  tmp.data_ptr(), tmp.numel(), what="first_order_edge_aware_loss")
        ctx.save_for_backward(d, i)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        d, i = ctx.saved_tensors
        (Cd, H, W), Ci = d.shape, i.shape[0]
        g = _lib.f32(g)
        dd = torch.empty_like(d) if ctx.needs_input_grad[0] else None
        di = torch.empty_like(i) if ctx.needs_input_grad[1] else None
        _lib.call("r3dg_edge_aware_backward", d.device, Cd, Ci, H, W, d.data_ptr(), i.data_ptr(), g.data_ptr(),
                  _lib.ptr(dd), _lib.ptr(di), what="first_order_edge_aware_loss backward")
        return dd, di


def first_order_edge_aware_loss(data, img):
    """Drop-in for utils/loss_utils.py:104: mean over [C,H,W] of sum_d |S_d(data)| * exp(-|S_d(img)|), S_d the
    normalised Sobel responses with replicate padding (kornia spatial_gradient).  data [Cd,H,W] and img [Ci,H,W] are
    float32 CUDA tensors; Cd and Ci are each 1 or C = max(Cd, Ci) (torch broadcasting).  Returns a 0-dim tensor;
    gradients flow to both inputs."""
    fn = "first_order_edge_aware_loss"
    for name, t in (("data", data), ("img", img)):
        _check_cuda_f32(fn, name, t)
        if t.dim() != 3:
            raise ValueError(f"{fn}: {name} must be [C,H,W] (got {tuple(t.shape)})")
    if data.shape[1:] != img.shape[1:]:
        raise ValueError(f"{fn}: image sizes differ: {tuple(data.shape)} vs {tuple(img.shape)}")
    Cd, Ci = data.shape[0], img.shape[0]
    if Cd != Ci and 1 not in (Cd, Ci):
        raise ValueError(f"{fn}: channel counts {Cd} and {Ci} do not broadcast")
    if data.device != img.device:
        raise ValueError(f"{fn}: inputs are on different devices ({data.device}, {img.device})")
    return _EdgeAware.apply(data, img)


class _TV(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        xc = _lib.f32(x)
        H, W = xc.shape[-2:]
        B = xc.numel() // (H * W)
        dev = xc.device
        out = torch.empty((), dtype=torch.float32, device=dev)
        tmp = _lib.scratch(max(_lib.load().r3dg_tv_tmp_bytes(B, H, W), 1), dev)
        _lib.call("r3dg_tv_forward", dev, B, H, W, xc.data_ptr(), out.data_ptr(), tmp.data_ptr(), tmp.numel(),
                  what="tv_loss")
        ctx.save_for_backward(xc)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (xc,) = ctx.saved_tensors
        H, W = xc.shape[-2:]
        B = xc.numel() // (H * W)
        g = _lib.f32(g)
        dx = torch.empty_like(xc)
        _lib.call("r3dg_tv_backward", xc.device, B, H, W, xc.data_ptr(), g.data_ptr(), dx.data_ptr(), what="tv_loss backward")
        return dx


def tv_loss(x):
    """Drop-in for utils/loss_utils.py:113: mean of the squared differences along dim -2 plus mean of those along
    dim -1, for a float32 CUDA tensor [..., H, W] with H, W >= 2 (non-contiguous views are fine).  Returns a 0-dim
    tensor."""
    _check_cuda_f32("tv_loss", "x", x)
    if x.dim() < 2:
        raise ValueError(f"tv_loss: x must be [..., H, W] (got {tuple(x.shape)})")
    if x.shape[-2] < 2 or x.shape[-1] < 2:
        # the reference returns NaN here (the mean of an empty difference tensor)
        raise ValueError(f"tv_loss: H and W must be at least 2 (got {tuple(x.shape)})")
    return _TV.apply(x)


_REGULARIZERS = {"first_order_edge_aware_loss": first_order_edge_aware_loss, "tv_loss": tv_loss}


def install(*modules, regularizers=False):
    """Rebind `ssim` in utils.loss_utils and in the modules that copied it with `from utils.loss_utils import ssim`
    (default: gaussian_renderer.render and gaussian_renderer.neilf); with regularizers=True also
    `first_order_edge_aware_loss` and `tv_loss` in the same modules.  Modules may be given as objects or names;
    names are imported.  Returns the modules rebound; `uninstall()` restores them."""
    fns = {"ssim": ssim, **(_REGULARIZERS if regularizers else {})}
    targets = []
    for m in (modules or DEFAULT_MODULES):
        if isinstance(m, str):
            __import__(m)
            m = sys.modules[m]
        targets.append(m)
    for m in targets:
        for name, fn in fns.items():
            _saved.append((m, name, m.__dict__.get(name)))
            setattr(m, name, fn)
    return targets


def uninstall():
    """Undo every `install()` in reverse order."""
    while _saved:
        m, name, prev = _saved.pop()
        setattr(m, name, prev)
