"""fp64 PyTorch restatement of the rasterizer's pseudo-normal / surface-xyz pass (csrc/composite.cu
surface_normal_kernel), differentiable with torch autograd: the truth of the surface-gradient tests."""
import numpy as np
import torch

EPS = float(np.float32(1e-7))          # the forward's max(opacity, 1e-7f)


def focal(W, H, tan_fovx, tan_fovy):
    """The kernels' fp32 focal lengths W / (2 tan_fovx), H / (2 tan_fovy)."""
    fx = np.float32(W) / (np.float32(2.0) * np.float32(tan_fovx))
    fy = np.float32(H) / (np.float32(2.0) * np.float32(tan_fovy))
    return float(fx), float(fy)


def _stencils(opacity, depth, W, H, tan_fovx, tan_fovy, cx, cy):
    o, dep = opacity.reshape(H, W), depth.reshape(H, W)
    dev, dt = o.device, o.dtype
    fx, fy = focal(W, H, tan_fovx, tan_fovy)
    d = dep / torch.where(o > EPS, o, torch.full_like(o, EPS))
    xs = torch.arange(W, device=dev, dtype=dt)
    ys = torch.arange(H, device=dev, dtype=dt)
    a = ((xs - float(np.float32(cx))) / fx)[None, :]
    b = ((ys - float(np.float32(cy))) / fy)[:, None]
    P = torch.stack([a * d, b * d, d])                                     # [3,H,W]
    xi, yi = torch.arange(W, device=dev), torch.arange(H, device=dev)
    xm, xp = (xi - 1).clamp(0, W - 1), (xi + 1).clamp(0, W - 1)
    ym, yp = (yi - 1).clamp(0, H - 1), (yi + 1).clamp(0, H - 1)
    at = lambda r, c: P[:, r][:, :, c]
    ga = 0.125 * (at(ym, xp) - at(ym, xm) + at(yp, xp) - at(yp, xm)) + 0.25 * (at(yi, xp) - at(yi, xm))
    gb = 0.125 * (at(yp, xm) - at(ym, xm) + at(yp, xp) - at(ym, xp)) + 0.25 * (at(yp, xi) - at(ym, xi))
    return P, ga, gb


def surface_normal(opacity, depth, viewmatrix, W, H, tan_fovx, tan_fovy, cx, cy):
    """opacity, depth [1,H,W] (or [H,W]), viewmatrix [4,4] (or [16]) -> (normal [3,H,W], surface_xyz [3,H,W]) in the
    dtype of the inputs.  normal_k = sum_i V[4k + i] N_i with N = -n / |n|, n = ga x gb (clamped-border Sobel stencils
    of the surface points), zero where !(|n| > 0)."""
    P, ga, gb = _stencils(opacity, depth, W, H, tan_fovx, tan_fovy, cx, cy)
    dt = P.dtype
    n = torch.linalg.cross(ga, gb, dim=0)
    sq = (n * n).sum(0)
    ok = sq > 0
    norm = torch.sqrt(torch.where(ok, sq, torch.ones_like(sq)))
    N = torch.where(ok, -n / norm, torch.zeros_like(n))
    M = viewmatrix.reshape(4, 4)[:3, :3].to(dt)                            # M[k][i] = V[4k + i]
    normal = torch.einsum("ki,ihw->khw", M, N)
    return normal, P


def ill_conditioned(opacity, depth, W, H, tan_fovx, tan_fovy, cx, cy, bound=1e7):
    """[H,W] bool: pixels whose normal is ill-conditioned, |n| > 0 but max|P| (|ga| + |gb|) > bound |n| over the
    pixel's 3x3 window.  There ga and gb are (nearly) parallel or cancel, e.g. on the background next to a silhouette
    where only one neighbour has a surface point: n is rounding noise of the stencil and dN/dn ~ 1/|n| is huge, so the
    exact derivative is not a meaningful yardstick for an implementation that associates the sums differently."""
    with torch.no_grad():
        P, ga, gb = _stencils(opacity.double(), depth.double(), W, H, tan_fovx, tan_fovy, cx, cy)
        n = torch.linalg.cross(ga, gb, dim=0)
        nn = n.norm(dim=0)
        pm = torch.nn.functional.max_pool2d(P.abs().amax(0)[None, None], 3, 1, 1)[0, 0]
        return (nn > 0) & (pm * (ga.norm(dim=0) + gb.norm(dim=0)) > bound * nn)
