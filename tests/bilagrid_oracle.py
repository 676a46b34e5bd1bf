"""fp64 truth of the bilateral-grid slice (relightable3dgaussian_b200/bilagrid.py, csrc/bilagrid.cu), two ways:

  slice64 / grads64   a numpy restatement with the analytic gradients: trilinear weights at
                      ix = (px + 0.5)(GX-1)/W, iy = (py + 0.5)(GY-1)/H, iz = luma (L-1), clamped to the grid (border);
                      dL/drgb = A^T g + [0 < iz < L-1] (L-1) (dL/diz) (0.299, 0.587, 0.114);
  torch_slice         F.grid_sample(align_corners=True, padding_mode="border") on grids[ids] plus the per-pixel 3x4
                      matmul, differentiated by autograd (in any dtype; fp32 on the GPU is the unfused formulation).

coords="fp64" computes the three coordinates in fp64.  coords="fp32" takes them as the kernel computes them in fp32:
ix = fl(fl(fl(px + 0.5) (GX-1)) / W) and iy likewise, luma = fma(0.114f, b, fma(0.587f, g, fl(0.299f r))) and
iz = fl(luma (L-1)), each step correctly rounded; cells, weights and everything after them stay fp64.  The kernel's
cells, weights (t = i - i0 is exact in fp32) and border flag are then exactly the oracle's, so the truth is continuous
around the kernel's coordinates and no pixel needs masking.  Both roundings matter: at W = 100003, GX = 1024 the fp32
ix is about an ulp (6e-5) away from the fp64 one, and luma's rounding times (L-1) moves iz by several of its ulps,
which puts the fp64-coordinate truth ~25 eps32 of the output's scale away at any shape.

scales64 gives, per output element, the magnitude each kernel result is rounded at: the sum of the absolute values of
the terms that make it.  A tolerance of a few ulps of that scale holds where terms cancel, and is exactly 0 where
nothing contributes.
"""
import numpy as np
import torch
import torch.nn.functional as F

LUMA = np.array([0.299, 0.587, 0.114])
LUMA32 = np.array([0.299, 0.587, 0.114], np.float32)
IDENTITY = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], np.float64)


def fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded.  a b is exact in fp64; the sum is rounded to odd (TwoSum gives its exact
    error), and a round-to-odd value with 53 >= 24 + 2 bits rounds to the nearest fp32 as the exact sum would."""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32)
    c = np.asarray(c, np.float32).astype(np.float64)
    s = p + c
    v = s - p
    e = (p - (s - v)) + (c - v)
    even = (np.ascontiguousarray(s).view(np.int64) & 1) == 0
    s = np.where((e != 0) & even, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def _axis(npix, n, coords="fp64"):
    if coords == "fp32":
        c = ((np.arange(npix, dtype=np.float32) + np.float32(0.5)) * np.float32(n - 1) / np.float32(npix))
        c = c.astype(np.float64)
    else:
        c = (np.arange(npix) + 0.5) / npix * (n - 1)
    i0 = np.minimum(np.floor(c).astype(np.int64), n - 2)
    return i0, c - i0


def z_coord(rgb, L, coords="fp64"):
    """(cell, weight, unclamped iz, inside) of the luma coordinate of rgb [..., 3, H, W] (channel axis -3)."""
    if coords == "fp32":
        r, g, b = np.moveaxis(np.asarray(rgb, np.float32), -3, 0)
        lum = fma32(LUMA32[2], b, fma32(LUMA32[1], g, LUMA32[0] * r))
        iz = (lum * np.float32(L - 1)).astype(np.float64)
    else:
        iz = np.tensordot(LUMA, np.moveaxis(rgb, -3, 0), axes=1) * (L - 1)
    c = np.clip(iz, 0, L - 1)
    z0 = np.minimum(np.floor(c).astype(np.int64), L - 2)
    return z0, c - z0, iz, (iz > 0) & (iz < L - 1)


def _corners(grid, rgb, coords="fp64"):
    """Per image: list of (xy weight [1|H,W], z weight [H,W], z index [H,W], y index [H,1], x index [1,W]) of the 8
    corners, the four of the lower z node first."""
    _, L, GY, GX = grid.shape
    _, H, W = rgb.shape
    x0, tx = _axis(W, GX, coords)
    y0, ty = _axis(H, GY, coords)
    z0, tz, _, _ = z_coord(rgb, L, coords)
    out = []
    for bz in (0, 1):
        wz = tz if bz else 1 - tz
        for by in (0, 1):
            wy = (ty if by else 1 - ty)[:, None]
            for bx in (0, 1):
                wx = (tx if bx else 1 - tx)[None, :]
                out.append((wx * wy, wz, z0 + bz, (y0 + by)[:, None], (x0 + bx)[None, :]))
    return out


def affine(grid, rgb, coords="fp64"):
    """A [12, H, W] of one image."""
    return sum(wxy * wz * grid[:, z, y, x] for wxy, wz, z, y, x in _corners(grid, rgb, coords))


def slice64(grids, rgb, ids, coords="fp64"):
    grids, rgb = np.asarray(grids, np.float64), np.asarray(rgb, np.float64)
    out = np.empty_like(rgb)
    for n, g in enumerate(ids):
        A = affine(grids[g], rgb[n], coords).reshape(3, 4, *rgb.shape[-2:])
        out[n] = np.einsum("cjhw,jhw->chw", A[:, :3], rgb[n]) + A[:, 3]
    return out


def _ext(x):
    return np.concatenate([x, np.ones_like(x[:1])])            # (r, g, b, 1)


def grads64(grids, rgb, ids, dout, coords="fp64"):
    """(dL/drgb [N,3,H,W], dL/dgrids [G,12,L,GY,GX], iz [N,H,W] unclamped) for the cotangent dout."""
    grids, rgb, dout = (np.asarray(a, np.float64) for a in (grids, rgb, dout))
    G, _, L, GY, GX = grids.shape
    drgb = np.empty_like(rgb)
    dgrids = np.zeros_like(grids)
    izs = []
    for n, g in enumerate(ids):
        x, d = rgb[n], dout[n]
        corners = _corners(grids[g], x, coords)
        A = sum(wxy * wz * grids[g][:, z, y, xx] for wxy, wz, z, y, xx in corners).reshape(3, 4, *x.shape[-2:])
        drgb[n] = np.einsum("cjhw,chw->jhw", A[:, :3], d)
        # dA/diz: the difference of the two bilinear luma slices around the pixel's z cell
        _, _, iz, inside = z_coord(x, L, coords)
        izs.append(iz)
        S = [sum(wxy * grids[g][:, z, y, xx] for wxy, _, z, y, xx in corners[4 * bz:4 * bz + 4]) for bz in (0, 1)]
        D = (S[1] - S[0]).reshape(3, 4, *x.shape[-2:])
        diz = np.einsum("cjhw,jhw,chw->hw", D[:, :3], x, d) + np.einsum("chw,chw->hw", D[:, 3], d)
        drgb[n] += np.where(inside, diz * (L - 1), 0.0)[None] * LUMA[:, None, None]
        u = np.einsum("chw,jhw->cjhw", d, _ext(x)).reshape(12, *x.shape[-2:])
        for wxy, wz, z, y, xx in corners:
            node = ((z * GY + y) * GX + xx).ravel()
            w = wxy * wz
            for k in range(12):
                dgrids[g, k] += np.bincount(node, weights=(w * u[k]).ravel(), minlength=L * GY * GX).reshape(L, GY, GX)
    return drgb, dgrids, np.stack(izs)


def scales64(grids, rgb, ids, dout, coords="fp64"):
    """Per-element scales (m_out [N,3,H,W], m_drgb [N,3,H,W], m_dgrids [G,12,L,GY,GX]): the sums of |term| of
      out_c       = sum over corners, j in (r, g, b, 1) of w grid[4c+j] x_j;
      dL/drgb_j   = sum over corners, c of w grid[4c+j] dout_c, plus where the luma term applies
                    0.299|0.587|0.114 (L-1) sum over corners, c, k of wxy grid[4c+k] x_k dout_c (dA/diz weighs a
                    corner by its xy weight: the z weight's derivative is -1 or +1);
      dL/dgrids   = sum over the (pixel, corner) pairs that reach the coefficient of w dout_c x_j.
    Corner magnitudes, not |A|: the kernel's nested lerps round at the scale of the node values, which can cancel to a
    small A."""
    grids, rgb, dout = (np.asarray(a, np.float64) for a in (grids, rgb, dout))
    G, _, L, GY, GX = grids.shape
    N, _, H, W = rgb.shape
    m_out, m_drgb = np.zeros_like(rgb), np.zeros_like(rgb)
    m_dgrids = np.zeros_like(grids)
    for n, g in enumerate(ids):
        x, d = _ext(np.abs(rgb[n])), np.abs(dout[n])
        _, _, _, inside = z_coord(rgb[n], L, coords)
        lz = 0.0
        for wxy, wz, z, y, xx in _corners(grids[g], rgb[n], coords):
            a = np.abs(grids[g][:, z, y, xx]).reshape(3, 4, H, W)
            w = wxy * wz
            m_out[n] += w * np.einsum("cjhw,jhw->chw", a, x)
            m_drgb[n] += w * np.einsum("cjhw,chw->jhw", a[:, :3], d)
            lz = lz + wxy * np.einsum("cjhw,jhw,chw->hw", a, x, d)
            node = ((z * GY + y) * GX + xx).ravel()
            u = np.einsum("chw,jhw->cjhw", d, x).reshape(12, H, W)
            for k in range(12):
                m_dgrids[g, k] += np.bincount(node, weights=(w * u[k]).ravel(), minlength=L * GY * GX).reshape(L, GY, GX)
        m_drgb[n] += np.where(inside, lz * (L - 1), 0.0)[None] * LUMA[:, None, None]
    return m_out, m_drgb, m_dgrids


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
