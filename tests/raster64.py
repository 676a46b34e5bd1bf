"""fp64 truth of the sums the rasterizer's backward compositor forms per Gaussian, on the kernel's own forward state.

The compositor adds, for every (pixel, contributor) pair, one term per gradient-row slot into the contributor's row.
Here the same pairs are taken from the kernel's forward (point_list, ranges, n_contrib, means2D, conic_opacity), every
pixel is recomposited in fp64 and each pair's terms are formed explicitly and index-added into two fp64 results per
row: g64, the signed sum (the row's gradient), and m_row, the sum of the terms' magnitudes (the row's scale).  A
kernel's fp32 row is then held to |g - g64| <= tau * m_row: per row, so faint rows count as much as bright ones, and
independent of the cotangent scale.

The kernel's discrete decisions are taken as given and re-checked in fp64: power > 0, alpha < 1/255, the 0.99 clamp and
the T (1 - alpha) < 1e-4 cut-off.  A pixel with any of them within AMBIGUOUS relative of its threshold (power: of the
magnitude of its terms) is ambiguous: an fp32 / fp64 flip there is no error.  The caller gives such pixels zero
cotangents, in the kernel's call and here alike, so that they add nothing to any row.

Outputs (those of a colors_precomp + cov3D_precomp call): dL_dcolors, dL_dfeatures and dL_dopacity as the row holds
them; dL_dmeans2D in the units the kernel writes (0.5 W, 0.5 H per pixel); dL_dcov3D through the fp64 projection of
cov3D to the conic (aa_oracle.cov2d and the 0.3 px^2 dilation).  dL/dalpha of a pair comes from autograd of the fp64
composite with alpha as a leaf; dalpha / d(mean2D, conic, opacity) is the closed form the reference differentiates
(alpha = opacity G, G = exp(power): the 0.99 clamp is not differentiated)."""
import torch

import aa_oracle

TILE = 16
AMBIGUOUS = 1e-4
T_CUT = 1e-4


def cov3d_jacobian(means3D, cov6, viewmatrix, W, H, tanfovx, tanfovy):
    """d(conic a, b, c) / d(cov3D six) of every Gaussian, [P,3,6] fp64 (the conic of cov2D + 0.3 I)."""
    six = cov6.detach().double().requires_grad_(True)
    a0, b, c0 = aa_oracle.cov2d(means3D.double(), aa_oracle.cov3d_from_six(six), viewmatrix.double(), W, H,
                                tanfovx, tanfovy)
    a, c = a0 + aa_oracle.DILATION, c0 + aa_oracle.DILATION
    det = a * c - b * b
    conic = (c / det, -b / det, a / det)
    rows = [torch.autograd.grad(k.sum(), six, retain_graph=True)[0] for k in conic]
    return torch.stack(rows, 1)


class Walk:
    """The pairs of one batch of tiles: pixels [n] by list positions [L] (L: the batch's largest n_contrib)."""

    def __init__(self, st, tiles, W, H):
        dev = st["means2D"].device
        gx = (W + TILE - 1) // TILE
        t = torch.as_tensor(tiles, device=dev)
        i = torch.arange(TILE * TILE, device=dev)
        px = ((t % gx)[:, None] * TILE + i % TILE).reshape(-1)
        py = ((t // gx)[:, None] * TILE + i // TILE).reshape(-1)
        tile = t[:, None].expand(-1, TILE * TILE).reshape(-1)
        keep = (px < W) & (py < H)
        self.px, self.py, tile = px[keep], py[keep], tile[keep]
        self.pix = self.py * W + self.px
        nc = st["n_contrib"].reshape(-1)[self.pix].long()
        self.nc = nc
        L = int(nc.max()) if nc.numel() else 0
        j = torch.arange(L, device=dev)
        self.inlist = j[None, :] < nc[:, None]
        lo = st["ranges"][tile, 0].long()
        pos = (lo[:, None] + j[None, :]).clamp_max(st["point_list"].numel() - 1)
        self.ids = torch.where(self.inlist, st["point_list"][pos].long(), torch.zeros_like(pos))
        m2 = st["means2D"].double()[self.ids]
        co = st["conic_opacity"].double()[self.ids]
        self.dx = m2[..., 0] - self.px.double()[:, None]
        self.dy = m2[..., 1] - self.py.double()[:, None]
        ca, cb, cc, self.op = co.unbind(-1)
        self.ca, self.cb, self.cc = ca, cb, cc
        self.power = -0.5 * (ca * self.dx ** 2 + cc * self.dy ** 2) - cb * self.dx * self.dy
        self.G = torch.exp(self.power.clamp_max(0.0))
        raw = self.op * self.G
        alpha = raw.clamp_max(0.99)
        self.valid = self.inlist & (self.power <= 0) & (alpha >= 1.0 / 255.0)
        self.alpha = torch.where(self.valid, alpha, torch.zeros_like(alpha))
        one = 1.0 - self.alpha
        T = torch.cumprod(torch.cat([torch.ones_like(one[:, :1]), one], 1), 1)
        self.T = T[:, :-1]
        self.T_final = T[:, -1]
        rel = lambda x, thr: (x / thr - 1.0).abs() <= AMBIGUOUS          # noqa: E731
        # power > 0 is the sign of a sum: ambiguous relative to the magnitude of its terms
        pterms = 0.5 * (ca.abs() * self.dx ** 2 + cc.abs() * self.dy ** 2) + (cb * self.dx * self.dy).abs()
        crit = {"power": self.inlist & (self.power.abs() < AMBIGUOUS * pterms),
                "alpha": self.inlist & rel(alpha, 1.0 / 255.0),
                "clamp": self.inlist & rel(raw, 0.99),
                "cut-off": self.valid & rel(self.T * one, T_CUT)}
        self.criteria = {k: v.any(1) for k, v in crit.items()}
        self.ambiguous = torch.stack(list(self.criteria.values())).any(0)
        # the kernel's n_contrib: its last contributor composites in fp64, and nothing before it reaches the cut-off
        last = (nc - 1).clamp_min(0)
        last_ok = (nc == 0) | self.valid.gather(1, last[:, None])[:, 0]
        early = (self.valid & (self.T * one < T_CUT)).any(1)
        self.nc_ok = last_ok & ~early

    def composite(self, st, bg, S, alpha):
        """fp64 images of the batch's pixels [n, 3 + 1 + 1 + S] (color, opacity, depth, features) for alpha [n, L]."""
        one = 1.0 - alpha
        T = torch.cumprod(torch.cat([torch.ones_like(one[:, :1]), one], 1), 1)
        w = alpha * T[:, :-1]
        rgb = st["rgb"].double()[self.ids]
        col = (w[..., None] * rgb).sum(1) + T[:, -1:] * bg.double()[None, :]
        opa = w.sum(1, keepdim=True)
        dep = (w * st["depths"].double()[self.ids]).sum(1, keepdim=True)
        parts = [col, opa, dep]
        if S:
            parts.append((w[..., None] * st["features"].double()[self.ids]).sum(1))
        return torch.cat(parts, 1)


def row_truth(st, walks, cots, bg, W, H, S, jac=None):
    """g64 and m_row of every output over the pairs of `walks`: {name: (g64 [P,k], m_row [P,k])}.  cots: the four
    cotangent planes (color [3,H,W], opacity [1,H,W], depth [1,H,W], feature [S,H,W]) of the backward call."""
    P = st["means2D"].shape[0]
    dev = st["means2D"].device
    planes = torch.cat([c.reshape(c.shape[0], -1) for c in cots if c.numel()], 0).double()    # [3 + 2 + S, HW]
    width = {"dL_dcolors": 3, "dL_dfeatures": S, "dL_dopacity": 1, "dL_dmeans2D": 2, "dL_dcov3D": 6}
    out = {k: (torch.zeros(P, n, dtype=torch.float64, device=dev), torch.zeros(P, n, dtype=torch.float64, device=dev))
           for k, n in width.items() if n}
    for wk in walks:
        cot = planes[:, wk.pix].T                                                        # [n, 5 + S]
        a = wk.alpha.clone().requires_grad_(True)
        img = wk.composite(st, bg, S, a)
        dA, = torch.autograd.grad((img * cot).sum(), a)
        v = wk.valid
        w = (wk.alpha * wk.T)[v]
        ids = wk.ids[v]
        ccol = w[:, None] * cot[:, :3][:, None, :].expand(-1, v.shape[1], -1)[v]
        terms = {"dL_dcolors": ccol, "dL_dopacity": (dA * wk.G)[v][:, None]}
        if S:
            terms["dL_dfeatures"] = w[:, None] * cot[:, 5:][:, None, :].expand(-1, v.shape[1], -1)[v]
        dpow = (dA * wk.op * wk.G)[v]
        dx, dy = wk.dx[v], wk.dy[v]
        ca, cb, cc = wk.ca[v], wk.cb[v], wk.cc[v]
        terms["dL_dmeans2D"] = torch.stack([dpow * -(ca * dx + cb * dy) * (0.5 * W),
                                            dpow * -(cc * dy + cb * dx) * (0.5 * H)], 1)
        # a term that is itself a sum of products counts the magnitudes of its products
        mags = {"dL_dmeans2D": dpow.abs()[:, None] * torch.stack([((ca * dx).abs() + (cb * dy).abs()) * (0.5 * W),
                                                                   ((cc * dy).abs() + (cb * dx).abs()) * (0.5 * H)], 1)}
        if jac is not None:
            dconic = torch.stack([-0.5 * dx * dx, -dx * dy, -0.5 * dy * dy], 1) * dpow[:, None]
            J = jac[ids]
            terms["dL_dcov3D"] = torch.einsum("nk,nks->ns", dconic, J)
            mags["dL_dcov3D"] = torch.einsum("nk,nks->ns", dconic.abs(), J.abs())
        for k, t in terms.items():
            out[k][0].index_add_(0, ids, t)
            out[k][1].index_add_(0, ids, mags.get(k, t).abs())
    return out


def walks_of(st, W, H, batch_pixels=1 << 14):
    """The Walks of every tile, batched so that one batch holds about `batch_pixels` pixels."""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    per = max(1, batch_pixels // (TILE * TILE))
    return [Walk(st, list(range(t0, min(t0 + per, gx * gy))), W, H) for t0 in range(0, gx * gy, per)]
