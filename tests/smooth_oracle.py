"""TEST INFRASTRUCTURE — not product code.

Seeded inputs (`smooth_case`, `tv_case`) and a PyTorch restatement of the reference's smoothness
regularisers (utils/loss_utils.py:104-105,113-117): kornia 0.6.12's `spatial_gradient(x, order=1)`
(Sobel kernel divided by sum |k| = 8, replicate padding of 1, [B,C,2,H,W]) as a replicate pad plus a
grouped convolution, `first_order_edge_aware_loss` and `tv_loss`, in fp32 or fp64, with IEEE
convolutions by default.  Parity status: PINNED against tests/golden/smooth.npz, which holds outputs
and autograd gradients of the reference's own function bodies executed on CPU in fp32 and fp64 on top
of this `spatial_gradient` (tests/golden/make_golden_smooth.py).  The GPU tests use it as the reference
formula at sizes the fixture cannot hold.
"""
import contextlib

import torch
import torch.nn.functional as F

from ssim_oracle import ieee_convolutions

# (name, kind, Cd, Ci, H, W, seed) of every edge-aware record in tests/golden/smooth.npz
EDGE_CASES = [
    ("pair33", "rendered", 3, 3, 24, 32, 0),
    ("pair13", "rendered", 1, 3, 24, 32, 1),
    ("pair31", "rendered", 3, 1, 24, 32, 2),
    ("pair11", "rendered", 1, 1, 24, 32, 3),
    ("masked", "masked", 3, 3, 40, 48, 4),
    ("masked13", "masked", 1, 3, 40, 48, 5),
    ("diffuse_normal", "normal", 3, 3, 32, 40, 6),
    ("constdata", "constdata", 3, 3, 24, 32, 7),
    ("constimg", "constimg", 3, 3, 24, 32, 8),
    ("hdr_img", "hdr", 3, 3, 24, 32, 9),
    ("px_1x1", "rendered", 3, 3, 1, 1, 10),
    ("row_1x17", "rendered", 3, 3, 1, 17, 11),
    ("col_13x1", "rendered", 1, 3, 13, 1, 12),
    ("tiny_2x2", "rendered", 3, 1, 2, 2, 13),
    ("tiny_3x5", "rendered", 3, 3, 3, 5, 14),
    ("strip_13x200", "rendered", 3, 3, 13, 200, 15),
]

# (name, shape, permuted, seed) of every TV record; `permuted` cases are x.permute(2, 0, 1) of an [H,W,C] tensor,
# as gaussian_renderer/neilf.py:306 passes env[0].permute(2, 0, 1)
TV_CASES = [
    ("env_permuted", (3, 16, 32), True, 0),
    ("img_3x24x32", (3, 24, 32), False, 1),
    ("batch_2x3x5x7", (2, 3, 5, 7), False, 2),
    ("min_1x2x2", (1, 2, 2), False, 3),
    ("strip_3x13x200", (3, 13, 200), False, 4),
]


def _rendered(C, H, W, g):
    """Piecewise-smooth shading with hard-edged discs and 2 % noise, in [0, 1]."""
    yy = torch.linspace(-1, 1, H).view(H, 1)
    xx = torch.linspace(-1, 1, W).view(1, W)
    a = torch.full((C, H, W), 0.1)
    for _ in range(6):
        cx, cy, r = (torch.rand(3, generator=g) * torch.tensor([1.6, 1.6, 0.5]) - torch.tensor([0.8, 0.8, -0.1])).tolist()
        col = torch.rand(C, 1, 1, generator=g)
        disc = (((xx - cx) ** 2 + (yy - cy) ** 2) < r * r).float()
        a = a * (1 - disc) + disc * col * (0.6 + 0.4 * torch.cos(3 * xx + 2 * yy))
    return (a + 0.02 * torch.randn(C, H, W, generator=g)).clamp(0, 1)


def _mask(H, W, g):
    """Foreground disc (image_mask of the stage-2 call sites) with two exactly constant patches cut out of it."""
    yy = torch.linspace(-1, 1, H).view(H, 1)
    xx = torch.linspace(-1, 1, W).view(1, W)
    m = ((xx ** 2 + yy ** 2) < 0.7).float()
    return m, (slice(H // 5, H // 5 + max(H // 4, 1)), slice(W // 2, W // 2 + max(W // 4, 1)))


def smooth_case(kind, Cd, Ci, H, W, seed):
    """(data [Cd,H,W], img [Ci,H,W], cotangent) on CPU, float32."""
    g = torch.Generator().manual_seed(9000 + seed)
    C = max(Cd, Ci)
    if kind == "rendered":                 # rendered attribute vs GT image
        d, i = _rendered(Cd, H, W, g), _rendered(Ci, H, W, g)
    elif kind == "masked":                 # render * image_mask, with constant patches in data and img: sign(0)
        m, patch = _mask(H, W, g)
        d = _rendered(Cd, H, W, g) * m
        d[:, patch[0], patch[1]] = 0.37
        i = _rendered(Ci, H, W, g)
        i[:, H // 10:H // 10 + max(H // 8, 3), W // 10:W // 10 + max(W // 8, 3)] = 0.5
    elif kind == "normal":                 # diffuse * mask vs a rendered normal in [-1, 1] (neilf.py:299)
        m, _ = _mask(H, W, g)
        d = _rendered(Cd, H, W, g) * m
        n = torch.nn.functional.normalize(_rendered(Ci, H, W, g) * 2 - 1 + torch.tensor([0.0, 0.0, 0.5]).view(-1, 1, 1)[:Ci], dim=0)
        i = n * m
    elif kind == "constdata":              # L = 0 and zero gradients, exactly
        d, i = torch.full((Cd, H, W), 0.3), _rendered(Ci, H, W, g)
    elif kind == "constimg":               # exp(-|S I|) = 1 everywhere
        d, i = _rendered(Cd, H, W, g), torch.full((Ci, H, W), 0.6)
    elif kind == "hdr":                    # img in [0, 50]: exp(-|S I|) spans many decades
        d, i = _rendered(Cd, H, W, g), 50.0 * _rendered(Ci, H, W, g)
    else:
        raise ValueError(kind)
    cot = 0.5 + torch.rand((), generator=g)
    assert d.shape[0] in (1, C) and i.shape[0] in (1, C)
    return d.float().contiguous(), i.float().contiguous(), cot


def tv_case(shape, permuted, seed):
    """(x, cotangent) on CPU, float32; x is a non-contiguous permute view when `permuted`."""
    g = torch.Generator().manual_seed(9500 + seed)
    if permuted:
        C, H, W = shape
        x = torch.rand(H, W, C, generator=g).permute(2, 0, 1)
    else:
        x = torch.rand(shape, generator=g)
    return x, 0.5 + torch.rand((), generator=g)


def sobel_kernel(dtype=torch.float32):
    """kornia get_sobel_kernel2d normalised: [[-1,0,1],[-2,0,2],[-1,0,1]] and its transpose, / 8."""
    kx = torch.tensor([[-1.0, 0.0, 1.0], [-2.0, 0.0, 2.0], [-1.0, 0.0, 1.0]])
    k = torch.stack([kx, kx.t()])
    return (k / k.abs().sum(dim=(-1, -2), keepdim=True)).to(dtype)


def spatial_gradient(x, mode="sobel", order=1, normalized=True, ieee=True):
    """kornia.filters.spatial_gradient(x, 'sobel', order=1, normalized=True) for x [B,C,H,W]: [B,C,2,H,W] (d/dx, d/dy).
    ieee=False leaves the convolution to cuDNN's defaults (TF32 for fp32), as the reference runs it."""
    assert mode == "sobel" and order == 1 and normalized
    B, C, H, W = x.shape
    w = sobel_kernel().to(device=x.device, dtype=x.dtype).unsqueeze(1).repeat(C, 1, 1, 1)     # [2C,1,3,3]
    padded = F.pad(x, [1, 1, 1, 1], mode="replicate")
    with ieee_convolutions() if ieee else contextlib.nullcontext():
        out = F.conv2d(padded, w, groups=C)
    return out.view(B, C, 2, H, W)


def first_order_edge_aware_loss(data, img, ieee=True):
    sg = lambda t: spatial_gradient(t[None], order=1, ieee=ieee)
    return (sg(data)[0].abs() * torch.exp(-sg(img)[0].abs())).sum(1).mean()


def tv_loss(depth):
    h_tv = torch.square(depth[..., 1:, :] - depth[..., :-1, :]).mean()
    w_tv = torch.square(depth[..., :, 1:] - depth[..., :, :-1]).mean()
    return h_tv + w_tv


def value_and_grads(fn, inputs, cot, dtype):
    """(value, [dL/dinput ...]) of fn(*inputs) in `dtype`, L = value * cot.  The backward convolutions run in IEEE
    fp32 too."""
    xs = [t.detach().to(dtype).requires_grad_(True) for t in inputs]
    with ieee_convolutions():
        v = fn(*xs)
        (v * cot.to(v)).backward()
    return v.detach(), [x.grad for x in xs]
