"""fp64 truth of the bilateral-grid slice (relightable3dgaussian_b200/bilagrid.py, csrc/bilagrid.cu), two ways:

  slice64 / grads64   a numpy restatement with the analytic gradients: trilinear weights at
                      ix = (px + 0.5)(GX-1)/W, iy = (py + 0.5)(GY-1)/H, iz = luma (L-1), clamped to the grid (border);
                      dL/drgb = A^T g + [0 < iz < L-1] (L-1) (dL/diz) (0.299, 0.587, 0.114);
  torch_slice         F.grid_sample(align_corners=True, padding_mode="border") on grids[ids] plus the per-pixel 3x4
                      matmul, differentiated by autograd (in any dtype; fp32 on the GPU is the unfused formulation).
"""
import numpy as np
import torch
import torch.nn.functional as F

LUMA = np.array([0.299, 0.587, 0.114])
IDENTITY = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float64)


def _axis(npix, n):
    c = (np.arange(npix) + 0.5) / npix * (n - 1)
    i0 = np.minimum(np.floor(c).astype(np.int64), n - 2)
    return i0, c - i0


def z_coord(rgb, L):
    """(cell, weight, unclamped iz, inside) of the luma coordinate of rgb [..., 3, H, W] (channel axis -3)."""
    iz = np.tensordot(LUMA, np.moveaxis(rgb, -3, 0), axes=1) * (L - 1)
    c = np.clip(iz, 0, L - 1)
    z0 = np.minimum(np.floor(c).astype(np.int64), L - 2)
    return z0, c - z0, iz, (iz > 0) & (iz < L - 1)


def _corners(grid, rgb):
    """Per image: list of (weight [H,W], z index [H,W], y index [H,1], x index [1,W]) of the 8 corners."""
    _, L, GY, GX = grid.shape
    _, H, W = rgb.shape
    x0, tx = _axis(W, GX)
    y0, ty = _axis(H, GY)
    z0, tz, _, _ = z_coord(rgb, L)
    out = []
    for bz in (0, 1):
        wz = tz if bz else 1 - tz
        for by in (0, 1):
            wy = (ty if by else 1 - ty)[:, None]
            for bx in (0, 1):
                wx = (tx if bx else 1 - tx)[None, :]
                out.append((wx * wy * wz, z0 + bz, (y0 + by)[:, None], (x0 + bx)[None, :]))
    return out


def affine(grid, rgb):
    """A [12, H, W] of one image."""
    return sum(w * grid[:, z, y, x] for w, z, y, x in _corners(grid, rgb))


def slice64(grids, rgb, ids):
    grids, rgb = np.asarray(grids, np.float64), np.asarray(rgb, np.float64)
    out = np.empty_like(rgb)
    for n, g in enumerate(ids):
        A = affine(grids[g], rgb[n]).reshape(3, 4, *rgb.shape[-2:])
        out[n] = np.einsum("cjhw,jhw->chw", A[:, :3], rgb[n]) + A[:, 3]
    return out


def grads64(grids, rgb, ids, dout):
    """(dL/drgb [N,3,H,W], dL/dgrids [G,12,L,GY,GX], iz [N,H,W] unclamped) for the cotangent dout."""
    grids, rgb, dout = (np.asarray(a, np.float64) for a in (grids, rgb, dout))
    G, _, L, GY, GX = grids.shape
    drgb = np.empty_like(rgb)
    dgrids = np.zeros_like(grids)
    izs = []
    for n, g in enumerate(ids):
        x, d = rgb[n], dout[n]
        A = affine(grids[g], x).reshape(3, 4, *x.shape[-2:])
        drgb[n] = np.einsum("cjhw,chw->jhw", A[:, :3], d)
        # dA/diz: the difference of the two bilinear luma slices around the pixel's z cell
        z0, _, iz, inside = z_coord(x, L)
        izs.append(iz)
        S = [0, 0]
        x0, tx = _axis(x.shape[2], GX)
        y0, ty = _axis(x.shape[1], GY)
        for bz in (0, 1):
            acc = 0
            for by in (0, 1):
                wy = (ty if by else 1 - ty)[:, None]
                for bx in (0, 1):
                    wx = (tx if bx else 1 - tx)[None, :]
                    acc = acc + wx * wy * grids[g][:, z0 + bz, (y0 + by)[:, None], (x0 + bx)[None, :]]
            S[bz] = acc
        D = (S[1] - S[0]).reshape(3, 4, *x.shape[-2:])
        diz = np.einsum("cjhw,jhw,chw->hw", D[:, :3], x, d) + np.einsum("chw,chw->hw", D[:, 3], d)
        drgb[n] += np.where(inside, diz * (L - 1), 0.0)[None] * LUMA[:, None, None]
        ext = np.concatenate([x, np.ones_like(x[:1])])            # (r, g, b, 1)
        u = np.einsum("chw,jhw->cjhw", d, ext).reshape(12, *x.shape[-2:])
        for w, z, y, xx in _corners(grids[g], x):
            node = ((z * GY + y) * GX + xx).ravel()
            for k in range(12):
                dgrids[g, k] += np.bincount(node, weights=(w * u[k]).ravel(), minlength=L * GY * GX).reshape(L, GY, GX)
    return drgb, dgrids, np.stack(izs)


def torch_slice(grids, rgb, ids):
    """The grid_sample formulation: grids [G,12,L,GY,GX], rgb [N,3,H,W] (any float dtype, any device)."""
    N, _, H, W = rgb.shape
    dt, dev = rgb.dtype, rgb.device
    xs = (torch.arange(W, dtype=dt, device=dev) + 0.5) / W
    ys = (torch.arange(H, dtype=dt, device=dev) + 0.5) / H
    lum = 0.299 * rgb[:, 0] + 0.587 * rgb[:, 1] + 0.114 * rgb[:, 2]
    gx, gy = xs[None, :].expand(H, W), ys[:, None].expand(H, W)
    coords = torch.stack([(2 * gx - 1).expand(N, H, W), (2 * gy - 1).expand(N, H, W), 2 * lum - 1], dim=-1)
    idx = torch.as_tensor(ids, dtype=torch.long, device=dev)
    A = F.grid_sample(grids[idx], coords[:, None], mode="bilinear", padding_mode="border", align_corners=True)
    A = A[:, :, 0].reshape(N, 3, 4, H, W)
    return (A[:, :, :3] * rgb[:, None]).sum(2) + A[:, :, 3]


def random_case(G, N, H, W, L=8, GY=16, GX=16, seed=0, luma_lo=0.0, luma_hi=1.0, noise=0.1):
    """Grids near the identity and images whose luma spans [luma_lo, luma_hi] (fp32 values, fp32 arrays)."""
    rs = np.random.default_rng(seed)
    grids = IDENTITY.reshape(1, 12, 1, 1, 1) + noise * rs.standard_normal((G, 12, L, GY, GX))
    rgb = rs.uniform(luma_lo, luma_hi, (N, 3, H, W))
    return grids.astype(np.float32), rgb.astype(np.float32)


def near_node_mask(iz, L, tol=1e-5):
    """Pixels whose luma coordinate lies within tol of a node or of the clamp bounds, where dL/drgb jumps."""
    return np.abs(iz - np.round(np.clip(iz, 0, L - 1))) < tol
