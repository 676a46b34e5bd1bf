"""TEST INFRASTRUCTURE — not product code.

Seeded SSIM inputs (`ssim_case`) and a PyTorch restatement of the reference's SSIM
(utils/loss_utils.py:20-63: `gaussian`, `create_window`, `_ssim`) that runs in fp32 or fp64 with
TF32 convolutions off.  Parity status: PINNED against tests/golden/ssim.npz, which holds outputs
and autograd gradients of the reference's own function bodies executed on CPU in fp32 and fp64
(tests/golden/make_golden_ssim.py).  The GPU tests use it as the reference formula at sizes the
fixture cannot hold.
"""
import contextlib
from math import exp

import torch
import torch.nn.functional as F

# (name, kind, shape, size_average, seed) of every record in tests/golden/ssim.npz
GOLDEN_CASES = [
    ("uniform", "uniform", (3, 48, 64), True, 0),
    ("close", "close", (3, 24, 32), True, 1),
    ("smooth", "smooth", (3, 24, 32), True, 2),
    ("nearconst", "nearconst", (3, 24, 32), True, 3),
    ("hdr", "hdr", (3, 24, 32), True, 4),
    ("identical", "identical", (3, 24, 32), True, 5),
    ("tiny_3x5x7", "uniform", (3, 5, 7), True, 6),
    ("pixel_1x1x1", "uniform", (1, 1, 1), True, 7),
    ("strip_3x13x200", "close", (3, 13, 200), True, 8),
    ("c1", "close", (1, 24, 32), True, 9),
    ("c4", "rendered", (4, 24, 32), True, 10),
    ("batch_mean", "close", (2, 3, 24, 40), True, 11),
    ("batch_per_image", "close", (2, 3, 24, 40), False, 12),
]


def ssim_case(kind, shape, seed):
    """(img1, img2, cotangent) on CPU, float32.  The cotangent is [N] for 4-D shapes (used with
    size_average=False) and a scalar 1 otherwise."""
    g = torch.Generator().manual_seed(7000 + seed)
    rand = lambda: torch.rand(shape, generator=g)
    randn = lambda: torch.randn(shape, generator=g)
    H, W = shape[-2], shape[-1]
    if kind == "uniform":                  # independent noise: SSIM ~ 0
        a, b = rand(), rand()
    elif kind == "close":                  # image vs image + 1 % noise: SSIM ~ 1
        a = rand()
        b = a + 0.01 * randn()
    elif kind == "smooth":                 # smooth ramps + 1e-3 noise: E[x^2] - mu^2 cancels
        yy = torch.linspace(0, 1, H).view(H, 1)
        xx = torch.linspace(0, 1, W).view(1, W)
        ramp = (0.2 + 0.5 * xx + 0.3 * yy).expand(shape)
        a = ramp + 1e-3 * randn()
        b = 0.98 * ramp + 0.01 + 1e-3 * randn()
    elif kind == "nearconst":              # 0.5 + 1e-4 noise: variances far below C2
        a, b = 0.5 + 1e-4 * randn(), 0.5 + 1e-4 * randn()
    elif kind == "hdr":                    # HDR radiance in [0, 4]
        a = 4.0 * rand()
        b = (a + 0.2 * randn()).clamp(0.0, 4.0)
    elif kind == "identical":
        a = rand()
        b = a.clone()
    elif kind == "rendered":               # piecewise-smooth shading with hard edges vs a noisy, shifted copy
        yy = torch.linspace(-1, 1, H).view(H, 1)
        xx = torch.linspace(-1, 1, W).view(1, W)
        a = torch.zeros(shape)
        for _ in range(6):
            cx, cy, r = (torch.rand(3, generator=g) * torch.tensor([1.6, 1.6, 0.5]) - torch.tensor([0.8, 0.8, -0.1])).tolist()
            col = torch.rand(shape[:-2] + (1, 1), generator=g)
            disc = (((xx - cx) ** 2 + (yy - cy) ** 2) < r * r).float()
            a = a * (1 - disc) + disc * col * (0.6 + 0.4 * torch.cos(3 * xx + 2 * yy))
        a = (a + 0.02 * randn()).clamp(0, 1)
        b = (torch.roll(a, 1, dims=-1) * 0.95 + 0.03 * randn()).clamp(0, 1)
    else:
        raise ValueError(kind)
    cot = torch.randn(shape[0], generator=g) if len(shape) == 4 else torch.tensor(1.0)
    return a.float().contiguous(), b.float().contiguous(), cot


@contextlib.contextmanager
def ieee_convolutions():
    """cuDNN convolutions in IEEE fp32 (torch's default lets them run in TF32), restored on exit."""
    prev = torch.backends.cudnn.conv.fp32_precision
    torch.backends.cudnn.conv.fp32_precision = "ieee"
    try:
        yield
    finally:
        torch.backends.cudnn.conv.fp32_precision = prev


def gaussian(window_size, sigma):
    gauss = torch.tensor([exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                         dtype=torch.float32)
    return gauss / gauss.sum()


def create_window(window_size, channel):
    w1 = gaussian(window_size, 1.5).unsqueeze(1)
    w2 = w1.mm(w1.t()).float().unsqueeze(0).unsqueeze(0)
    return w2.expand(channel, 1, window_size, window_size).contiguous()


def ssim(img1, img2, window_size=11, size_average=True, dtype=None, ieee=True):
    """The reference's ssim, computed in `dtype` (default: the inputs' dtype).  As in the reference, the
    window is built in float32 and then cast to the compute type.  ieee=False leaves the convolutions to
    cuDNN's defaults (TF32 for fp32), as the reference runs them."""
    if dtype is not None:
        img1, img2 = img1.to(dtype), img2.to(dtype)
    channel = img1.size(-3)
    window = create_window(window_size, channel).to(device=img1.device, dtype=img1.dtype)
    pad = window_size // 2
    with ieee_convolutions() if ieee else contextlib.nullcontext():
        mu1 = F.conv2d(img1, window, padding=pad, groups=channel)
        mu2 = F.conv2d(img2, window, padding=pad, groups=channel)
        mu1_sq = mu1.pow(2)
        mu2_sq = mu2.pow(2)
        mu1_mu2 = mu1 * mu2
        sigma1_sq = F.conv2d(img1 * img1, window, padding=pad, groups=channel) - mu1_sq
        sigma2_sq = F.conv2d(img2 * img2, window, padding=pad, groups=channel) - mu2_sq
        sigma12 = F.conv2d(img1 * img2, window, padding=pad, groups=channel) - mu1_mu2
    C1 = 0.01 ** 2
    C2 = 0.03 ** 2
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    if size_average:
        return ssim_map.mean()
    return ssim_map.mean(1).mean(1).mean(1)


def value_and_grads(fn, a, b, cot, size_average, dtype):
    """(value, dL/da, dL/db) of fn(a, b, size_average) in `dtype`, L = <value, cot>.  The backward
    convolutions run in IEEE fp32 too."""
    a = a.detach().to(dtype).requires_grad_(True)
    b = b.detach().to(dtype).requires_grad_(True)
    with ieee_convolutions():
        v = fn(a, b, size_average)
        (v * cot.to(v)).sum().backward()
    return v.detach(), a.grad, b.grad
