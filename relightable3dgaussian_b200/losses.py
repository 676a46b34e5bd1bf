"""Fused D-SSIM loss with the signature and return shapes of the reference's
`ssim(img1, img2, window_size=11, size_average=True)` (utils/loss_utils.py:32-63), backed by the sm_90a kernels
r3dg_ssim_forward / _backward (csrc/ssim.cu).

The reference calls it every training step (gaussian_renderer/render.py:150; twice in
gaussian_renderer/neilf.py:227,234) and as an evaluation metric (eval_nvs.py:72,
eval_relighting_syn4.py:191,195).  Its callers import the name with `from utils.loss_utils import ssim`, so
`install()` rebinds it in utils.loss_utils and in every module that already holds a copy (a 2-line plug-in, see
INTEGRATION.md).

Differences from the reference, all deliberate: the result is computed in IEEE fp32 (cuDNN runs the reference's
convolutions in TF32 under torch's defaults), the reduction is deterministic, and ssim(x, x) is exactly 1.  Only
what the call sites use is supported; anything else raises instead of falling back to PyTorch.
"""
import sys

import torch
from torch.autograd.function import once_differentiable

from . import _lib

DEFAULT_MODULES = ("utils.loss_utils", "gaussian_renderer.render", "gaussian_renderer.neilf")
_saved = []            # (module, previous ssim) of every rebinding made by install()


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


class _SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2, size_average):
        lib = _lib.load()
        x, y = img1.detach().contiguous(), img2.detach().contiguous()
        N = 1 if x.dim() == 3 else x.shape[0]
        C, H, W = x.shape[-3:]
        dev = x.device
        out = torch.empty(() if size_average else (N,), dtype=torch.float32, device=dev)
        tmp = torch.empty(max(lib.r3dg_ssim_tmp_bytes(N, C, H, W), 1), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.r3dg_ssim_forward(N, C, H, W, x.data_ptr(), y.data_ptr(), int(size_average), out.data_ptr(),
                                             tmp.data_ptr(), tmp.numel(), _stream(dev)), "ssim")
        ctx.save_for_backward(x, y)
        ctx.size_average = size_average
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        lib = _lib.load()
        x, y = ctx.saved_tensors
        N = 1 if x.dim() == 3 else x.shape[0]
        C, H, W = x.shape[-3:]
        dev = x.device
        g = g.float().contiguous()
        grads = []
        for need, a, b in ((ctx.needs_input_grad[0], x, y), (ctx.needs_input_grad[1], y, x)):   # dL/dimg2: img1 <-> img2
            d = None
            if need:
                d = torch.empty_like(a)
                with torch.cuda.device(dev):
                    _lib.check(lib.r3dg_ssim_backward(N, C, H, W, a.data_ptr(), b.data_ptr(), int(ctx.size_average),
                                                      g.data_ptr(), d.data_ptr(), _stream(dev)), "ssim backward")
            grads.append(d)
        return grads[0], grads[1], None


def ssim(img1, img2, window_size=11, size_average=True):
    """Drop-in for utils/loss_utils.py:32: mean SSIM of two [C,H,W] or [N,C,H,W] float32 CUDA images (0-dim), or
    per image ([N]) when size_average is False on 4-D input.  Gradients flow to both inputs."""
    if window_size != 11:
        raise ValueError(f"ssim: only window_size=11 is supported (got {window_size})")
    for name, t in (("img1", img1), ("img2", img2)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError(f"ssim: {name} must be a CUDA tensor")
        if t.dtype != torch.float32:
            raise TypeError(f"ssim: {name} must be float32 (got {t.dtype})")
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


def install(*modules):
    """Rebind `ssim` in utils.loss_utils and in the modules that copied it with `from utils.loss_utils import ssim`
    (default: gaussian_renderer.render and gaussian_renderer.neilf).  Modules may be given as objects or names;
    names are imported.  Returns the modules rebound; `uninstall()` restores them."""
    targets = []
    for m in (modules or DEFAULT_MODULES):
        if isinstance(m, str):
            __import__(m)
            m = sys.modules[m]
        targets.append(m)
    for m in targets:
        _saved.append((m, m.__dict__.get("ssim")))
        m.ssim = ssim
    return targets


def uninstall():
    """Undo every `install()` in reverse order."""
    while _saved:
        m, prev = _saved.pop()
        m.ssim = prev
