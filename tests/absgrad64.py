"""fp64 truth of the absolute screen-space gradients (absgrad) the rasterizer's backward forms per Gaussian.

On the pairs of raster64.Walk (the kernel's own forward state, every pixel recomposited in fp64), each (pixel,
contributor) pair's two dL/dmean2D terms are formed as raster64.row_truth forms them, in the units the kernel writes
(0.5 W and 0.5 H per pixel).  Their magnitudes are index-added per row: absgrad64 [P,2].  The signed sums of the same
terms, g64 [P,2], come along for the invariants absgrad >= |g| (componentwise) and absgrad == |g| for a Gaussian that
one pixel composites.  Ambiguous pixels are handled by the caller as in raster64: zero cotangents."""
import torch

import raster64


def row_truth(st, walks, cots, bg, W, H, S):
    """(absgrad64 [P,2], g64 [P,2]) over the pairs of `walks`.  cots: the four cotangent planes (color [3,H,W], opacity
    [1,H,W], depth [1,H,W], feature [S,H,W]) of the backward call, as raster64.row_truth takes them."""
    P = st["means2D"].shape[0]
    dev = st["means2D"].device
    planes = torch.cat([c.reshape(c.shape[0], -1) for c in cots if c.numel()], 0).double()
    absg = torch.zeros(P, 2, dtype=torch.float64, device=dev)
    sig = torch.zeros(P, 2, dtype=torch.float64, device=dev)
    for wk in walks:
        cot = planes[:, wk.pix].T
        a = wk.alpha.clone().requires_grad_(True)
        img = wk.composite(st, bg, S, a)
        dA, = torch.autograd.grad((img * cot).sum(), a)
        v = wk.valid
        dpow = (dA * wk.op * wk.G)[v]
        dx, dy = wk.dx[v], wk.dy[v]
        ca, cb, cc = wk.ca[v], wk.cb[v], wk.cc[v]
        t = torch.stack([dpow * -(ca * dx + cb * dy) * (0.5 * W), dpow * -(cc * dy + cb * dx) * (0.5 * H)], 1)
        ids = wk.ids[v]
        absg.index_add_(0, ids, t.abs())
        sig.index_add_(0, ids, t)
    return absg, sig


def walks_of(st, W, H, batch_pixels=1 << 14):
    """raster64.walks_of without the batches in which no pixel has a contributor (a Walk needs one)."""
    gx, gy = (W + raster64.TILE - 1) // raster64.TILE, (H + raster64.TILE - 1) // raster64.TILE
    per = max(1, batch_pixels // (raster64.TILE * raster64.TILE))
    nc = st["n_contrib"].reshape(-1)
    out = []
    for t0 in range(0, gx * gy, per):
        tiles = list(range(t0, min(t0 + per, gx * gy)))
        t = torch.as_tensor(tiles, device=nc.device)
        i = torch.arange(raster64.TILE * raster64.TILE, device=nc.device)
        px = ((t % gx)[:, None] * raster64.TILE + i % raster64.TILE).reshape(-1)
        py = ((t // gx)[:, None] * raster64.TILE + i // raster64.TILE).reshape(-1)
        keep = (px < W) & (py < H)
        if bool((nc[(py * W + px)[keep]] > 0).any()):
            out.append(raster64.Walk(st, tiles, W, H))
    return out
