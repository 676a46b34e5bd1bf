"""One differentiable fp64 renderer of the rasterizer, on the kernel's own per-pixel lists: the truth of every mode and
mode combination at once.

The record of every Gaussian is raydepth64.record (proj64.record with the depth plane appended) under torch.func.vmap:
SH colours up to degree 3 with the kernel's `clamped` flags taken as given, the antialiasing opacity factor rho, the 3D
filter's dilation, cov3D_precomp, and the projection backward's conventions (frustum clamp, linearised conic inverse,
ndc = h / (w + 1e-7)).  viewmatrix, projmatrix and campos are tensors of the camera, so that they can be leaves.

The pixels' lists are indexed as raster64.Walk indexes them, from the kernel's point_list, ranges and n_contrib, a
batch of tiles at a time.  Each pixel composites front to back in fp64 with the forward's decisions re-taken in fp64
(power > 0, alpha < 1/255, the 0.99 clamp with the reference's derivative of alpha = o G, the stop at n_contrib):

    color, opacity, depth (the centre's tz, or with ray depth the plane tz - p . (mean2D - pixel)), the S features,
    depth2 = sum w d^2 and the median depth (d of the entry at the kernel's median position; depthstats64's rule
    without one), and from opacity and depth the pseudo-normal and surface_xyz (surface_oracle.surface_normal).

`off` [P,3], when the leaves hold it, is a zero leaf added to the projected mean (ndc x, ndc y) and to the composited
tz: its gradient is the kernel's dL_dmeans2D.  Every (pixel, entry) pair has a zero leaf of its own added to the
entry's projected mean in that pixel, in ndc units: its gradient is the pair's whole dL/dmean2D (the alpha term, the
ray-depth plane's -p dL/dd and the median's term alike), and absgrad() sums its magnitudes per Gaussian.  A third
component of the pair leaf is added to the entry's opacity in that pixel: opacity_magnitude() sums the magnitudes of
those terms, m_row of the opacity (raster64's row scale).

The pixels where fp32 and fp64 may decide differently are returned by criterion (`ambiguous`): raster64.Walk's alpha,
power, clamp and cut-off tests on the kernel's own means2D and conic, the median's T within depthstats64.AMBIGUOUS of
0.5, the ill-conditioned normals of surface_oracle, and the pixels that composite a row of proj64.ambiguous_rows.
The callers give those pixels zero cotangents, in the kernel's call and here alike."""
import torch
from torch.func import vmap

import absgrad64
import depthstats64
import proj64
import raydepth64
import surface_oracle


class Camera(proj64.Camera):
    """proj64.Camera with the principal point the pseudo-normal needs."""

    def __init__(self, viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy, cx, cy):
        super().__init__(viewmatrix, projmatrix, campos, W, H, tanfovx, tanfovy)
        self.cx, self.cy = float(cx), float(cy)


def record(leaves, const, cam, D=0, aa=False, f3d=False):
    """[P, 12] fp64 records (proj64.REC and the depth plane p x, p y), differentiable in the leaves and the camera."""
    names = [k for k in leaves if k != "off"]
    return vmap(lambda lv, cs: raydepth64.record(lv, cs, cam, D, aa=aa, f3d=f3d)[0])(
        {k: leaves[k] for k in names}, const)


class Render:
    """The images (`images`: name -> [C,H,W]), the pair leaves and the ambiguous pixels and rows of one render()."""

    def __init__(self, P, H, W):
        self.P, self.H, self.W = P, H, W
        self.images = {}
        self.pairs = []                  # (leaf [n,L,3], ids [n,L], composited [n,L]) per batch of tiles
        self.op_factor = None            # [P]: the composited opacity over the leaf's (rho, the 3D filter's coef)
        self.ambiguous = {}              # criterion -> [H,W] bool
        self.ambiguous_rows = {}         # criterion -> [P] bool
        self.median_pos = None           # [H,W], the fp64 rule's 1-based position (0: none)
        self.max_list = 0                # the longest n_contrib walked

    def pair_leaves(self):
        return [p[0] for p in self.pairs]

    def absgrad(self, grads):
        """absgrad64 [P,2]: per Gaussian, the sum of |dL/dmean2D| over its composited pairs (grads: the gradients of
        pair_leaves(), in order)."""
        dev = self.pairs[0][0].device if self.pairs else "cpu"
        out = torch.zeros(self.P, 2, dtype=torch.float64, device=dev)
        for (_, ids, keep), g in zip(self.pairs, grads):
            if g is not None:
                out.index_add_(0, ids[keep], g[keep][:, :2].abs())
        return out

    def opacity_magnitude(self, grads):
        """m_row [P] of the opacity leaf: the sum of the magnitudes of its pairs' terms (grads as absgrad's)."""
        out = torch.zeros(self.P, dtype=torch.float64, device=self.op_factor.device)
        for (_, ids, keep), g in zip(self.pairs, grads):
            if g is not None:
                out.index_add_(0, ids[keep], g[keep][:, 2].abs())
        return out * self.op_factor

    def ambiguous_pixels(self):
        """[H,W] bool: any criterion."""
        m = torch.zeros(self.H, self.W, dtype=torch.bool, device=next(iter(self.images.values())).device)
        for v in self.ambiguous.values():
            m |= v
        return m


def render(leaves, const, cam, st, bg, *, D=0, aa=False, f3d=False, ray_depth=False, depth_stats=False,
           surface=False, batch_pixels=1 << 14, shift=None):
    """fp64 outputs of one view on the kernel's lists.

    leaves: {means3D [P,3], opacities [P,1], scales [P,3] + rotations [P,4] or cov3D [P,6], shs [P,M,3] or colors
    [P,3], features [P,S], optionally off [P,3]} (fp64).  const: {clamped [P,3] with shs, filter_3d [P] with f3d}.
    cam: Camera.  st: the kernel's forward state {point_list, ranges, n_contrib [H,W], means2D, conic_opacity and, for
    the median, median_pos [H,W]} (raster64.Walk's).  bg [3].  shift: {(batch, pixel, entry): [2]}, constants added to
    those pair leaves' mean components (finite differences of a pair)."""
    W, H = cam.W, cam.H
    m3 = leaves["means3D"]
    P, dev = m3.shape[0], m3.device
    rec = record(leaves, const, cam, D, aa=aa, f3d=f3d)
    ndc, tz, conic, op, col, pl = rec[:, 0:2], rec[:, 2], rec[:, 3:6], rec[:, 6], rec[:, 7:10], rec[:, 10:12]
    if "off" in leaves:
        ndc, tz = ndc + leaves["off"][:, :2], tz + leaves["off"][:, 2]
    half = torch.tensor([0.5 * W, 0.5 * H], dtype=torch.float64, device=dev)
    mean2D = (ndc + 1.0) * half - 0.5
    feats = leaves["features"]
    S = feats.shape[1]
    ch = torch.cat([col, feats], 1)

    out = Render(P, H, W)
    out.op_factor = (op / leaves["opacities"].reshape(-1)).detach()
    row_crit = proj64.ambiguous_rows({k: v.detach() for k, v in leaves.items() if k != "off"},
                                     {k: v.detach() for k, v in const.items()}, cam_detached(cam), D, aa=aa, f3d=f3d)
    out.ambiguous_rows = row_crit
    amb_rows = torch.stack(list(row_crit.values())).any(0)
    crit = {k: torch.zeros(H * W, dtype=torch.bool, device=dev)
            for k in ("power", "alpha", "clamp", "cut-off", "median", "rows")}
    parts = {k: [] for k in ("color", "opacity", "depth", "feature", "depth2", "median")}
    pixels, mpos_all = [], []
    kpos = st.get("median_pos")
    for b, wk in enumerate(absgrad64.walks_of(st, W, H, batch_pixels)):
        ids, inl = wk.ids, wk.inlist
        out.max_list = max(out.max_list, int(wk.nc.max()))
        pair = torch.zeros(*ids.shape, 3, dtype=torch.float64, device=dev, requires_grad=True)
        moved = pair
        for (bb, i, j), v in (shift or {}).items():
            if bb == b:
                at = (torch.tensor([i], device=dev), torch.tensor([j], device=dev))
                moved = moved.index_put(at, torch.cat([torch.as_tensor(v, dtype=torch.float64, device=dev), torch.zeros(1, dtype=torch.float64, device=dev)])[None], accumulate=True)
        m = mean2D[ids] + moved[..., :2] * half
        dx = m[..., 0] - wk.px.double()[:, None]
        dy = m[..., 1] - wk.py.double()[:, None]
        A, B, C = conic[ids].unbind(-1)
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        raw = (op[ids] + moved[..., 2]) * torch.exp(power)
        alpha = raw - (raw - 0.99).clamp_min(0.0).detach()             # the clamp, with the derivative of o G
        keep = inl & (power <= 0) & (alpha >= 1.0 / 255.0)
        alpha = torch.where(keep, alpha, torch.zeros_like(alpha))
        one = 1.0 - alpha
        Tall = torch.cumprod(torch.cat([torch.ones_like(one[:, :1]), one], 1), 1)
        T, Tf = Tall[:, :-1], Tall[:, -1]
        w = alpha * T
        d = tz[ids] - pl[ids, 0] * dx - pl[ids, 1] * dy if ray_depth else tz[ids]
        c = torch.einsum("nl,nlc->nc", w, ch[ids])
        parts["color"].append(c[:, :3] + Tf[:, None] * bg[None, :])
        parts["feature"].append(c[:, 3:])
        parts["opacity"].append(w.sum(1))
        parts["depth"].append((w * d).sum(1))
        if depth_stats:
            d2, med, pos = depthstats64.stats(w, d, T, keep)
            if kpos is not None:
                k = kpos.reshape(-1)[wk.pix].long()
                med = torch.where(k > 0, d.gather(1, (k - 1).clamp_min(0)[:, None])[:, 0], torch.zeros_like(d2))
            parts["depth2"].append(d2)
            parts["median"].append(med)
            mpos_all.append(pos)
            crit["median"][wk.pix] = (keep & ((T.detach() - 0.5).abs() <= depthstats64.AMBIGUOUS)).any(1)
        for k, v in wk.criteria.items():
            crit[k][wk.pix] = v
        crit["rows"][wk.pix] = (keep & amb_rows[ids]).any(1)
        out.pairs.append((pair, ids, keep))
        pixels.append(wk.pix)

    pix = torch.cat(pixels) if pixels else torch.zeros(0, dtype=torch.long, device=dev)
    # pixels no batch walks (empty lists): background colour, zero elsewhere
    Tfull = torch.ones(H * W, dtype=torch.float64, device=dev)

    def image(name, width):
        img = torch.zeros(H * W, width, dtype=torch.float64, device=dev)
        if name == "color":
            img = img + bg[None, :] * Tfull[:, None]
        if parts[name]:
            v = torch.cat([p.reshape(p.shape[0], -1) for p in parts[name]])
            img = img.index_copy(0, pix, v)
        return img.T.reshape(width, H, W)

    out.images = dict(color=image("color", 3), opacity=image("opacity", 1), depth=image("depth", 1),
                      feature=image("feature", S))
    if depth_stats:
        out.images["depth2"] = image("depth2", 1)
        out.images["median"] = image("median", 1)
        mp = torch.zeros(H * W, dtype=torch.long, device=dev)
        if mpos_all:
            mp[pix] = torch.cat(mpos_all)
        out.median_pos = mp.view(H, W)
    if surface:
        n, xyz = surface_oracle.surface_normal(out.images["opacity"], out.images["depth"], cam.V, W, H, cam.tanfovx,
                                               cam.tanfovy, cam.cx, cam.cy)
        out.images["normal"], out.images["xyz"] = n, xyz
        crit["normal"] = surface_oracle.ill_conditioned(out.images["opacity"].detach(), out.images["depth"].detach(),
                                                        W, H, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy).reshape(-1)
    out.ambiguous = {k: v.view(H, W) for k, v in crit.items()}
    return out


def cam_detached(cam):
    """A copy of `cam` whose tensors carry no graph."""
    return Camera(cam.V.detach(), cam.P.detach(), cam.campos.detach(), cam.W, cam.H, cam.tanfovx, cam.tanfovy,
                  getattr(cam, "cx", 0.0), getattr(cam, "cy", 0.0))
