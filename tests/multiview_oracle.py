"""The multi-view consistency losses (include/r3dg_b200.h, r3dg_multiview_*) restated in PyTorch from their definition,
in any dtype and on any device.  Autograd through it gives the definition's gradients; in float64 it is the truth the
kernels are held to, and in float32 it measures the error an fp32 formulation makes on its own.  Also the scenes the
tests and tools/bench_multiview.py share: smooth random maps and an analytic tilted plane."""
import math

import torch
import torch.nn.functional as F

MIN_Z, NCC_EPS, MAX_COST = 1e-6, 1e-8, 0.9


class Cam:
    """A view's camera as the loss reads it: viewmatrix [4,4] (row-vector world -> camera) and the intrinsics."""

    def __init__(self, viewmatrix, tanfovx, tanfovy, cx, cy):
        self.viewmatrix, self.tanfovx, self.tanfovy, self.cx, self.cy = viewmatrix, tanfovx, tanfovy, cx, cy

    @staticmethod
    def of(settings):
        return Cam(settings.viewmatrix, settings.tanfovx, settings.tanfovy, settings.cx, settings.cy)

    def K(self, H, W, dtype):
        """(fx, fy, cx, cy) rounded to dtype, as the kernels round them (fx computed in double)."""
        r = lambda v: torch.tensor(v, dtype=dtype).item()
        return r(W / (2.0 * self.tanfovx)), r(H / (2.0 * self.tanfovy)), r(self.cx), r(self.cy)


def _safe(cond, x, fill=1.0):
    return torch.where(cond, x, torch.full_like(x, fill))


def bilinear(img, u, v):
    """img [H,W] at pixel coordinates (u, v): align corners, zero padding; outside [-1, W) x [-1, H) exactly 0."""
    H, W = img.shape
    ok = (u >= -1) & (u < W) & (v >= -1) & (v < H)
    u, v = _safe(ok, u, 0.0), _safe(ok, v, 0.0)
    x0, y0 = torch.floor(u), torch.floor(v)
    ax, ay = u - x0, v - y0
    bx, by = 1 - ax, 1 - ay
    ix, iy = x0.long(), y0.long()

    def tap(i, j):
        inb = (i >= 0) & (i < W) & (j >= 0) & (j < H) & ok
        return img[j.clamp(0, H - 1), i.clamp(0, W - 1)] * inb

    return bx * by * tap(ix, iy) + ax * by * tap(ix + 1, iy) + bx * ay * tap(ix, iy + 1) + ax * ay * tap(ix + 1, iy + 1)


def _grid(c, extent):
    """How far a sampling coordinate lies from the nearest grid line, in units of 2e-4 + 2e-6 |c| pixels (about 1700
    fp32 ulps at |c| = 1 and 2 at |c| = 4096): the bilinear sample's derivative jumps at a grid line, and the kernel's
    fp32 coordinate, through the reprojection or the plane homography, may lie on the other side when this is below
    1.  On an axis one pixel long, q and the warped taps are exact integers in the scenes that test such images:
    they are built with exact arithmetic (axis-aligned cameras, principal point 0, equal focal lengths), which fp32
    reproduces, so an exact integer there counts as decided."""
    c = c.detach()
    d = (c - torch.round(c)).abs() / (2e-4 + 2e-6 * c.abs())
    return torch.where((c == torch.round(c)) & (extent == 1), torch.full_like(d, float("inf")), d)


def _taps_le0(img, u, v):
    """How many of the bilinear taps of (u, v) that carry weight and lie in the image hold a value <= 0."""
    H, W = img.shape
    x0, y0 = torch.floor(u), torch.floor(v)
    ax, ay = u - x0, v - y0
    ix, iy = x0.long(), y0.long()
    n = torch.zeros_like(ix)
    for dx, dy, wt in ((0, 0, (1 - ax) * (1 - ay)), (1, 0, ax * (1 - ay)), (0, 1, (1 - ax) * ay), (1, 1, ax * ay)):
        i, j = ix + dx, iy + dy
        inb = (i >= 0) & (i < W) & (j >= 0) & (j < H) & (wt > 0)
        n = n + (inb & (img[j.clamp(0, H - 1), i.clamp(0, W - 1)] <= 0)).long()
    return n


def _pair(depth_r, depth_n, normal_r, gray_r, gray_n, cam_r, cam_n, tau, dtype, w=None):
    """Per-pixel terms of one pair: dict of geo / photo contributions and masks, with the decision quantities."""
    H, W = depth_r.shape
    dev = depth_r.device
    fxr, fyr, cxr, cyr = cam_r.K(H, W, dtype)
    fxn, fyn, cxn, cyn = cam_n.K(H, W, dtype)
    vr, vn = cam_r.viewmatrix.to(dev, dtype), cam_n.viewmatrix.to(dev, dtype)
    Rr, Rn, tr, tn = vr[:3, :3].T, vn[:3, :3].T, vr[3, :3], vn[3, :3]
    R = Rn @ Rr.T
    t = tn - R @ tr
    ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=dtype), torch.arange(W, device=dev, dtype=dtype),
                            indexing="ij")
    xs, ys = xs.reshape(-1), ys.reshape(-1)
    # a non-finite depth is never valid: +inf makes q (reference) or phi (neighbour tap) NaN, -inf fails D > 0.  They
    # are replaced by 0 where they are read, so that no inf * 0 reaches the gradients of the valid pixels.
    D_raw = depth_r.reshape(-1)
    D = torch.where(torch.isfinite(D_raw), D_raw, torch.zeros_like(D_raw))
    depth_nf = torch.where(torch.isfinite(depth_n), depth_n, torch.zeros_like(depth_n))
    u = torch.stack([(xs - cxr) / fxr, (ys - cyr) / fyr, torch.ones_like(xs)], -1)
    X = D[:, None] * u
    Y = X @ R.T + t
    ok = (D > 0) & (Y[:, 2] > MIN_Z)
    Yz = _safe(ok, Y[:, 2])
    qx, qy = fxn * (Y[:, 0] / Yz) + cxn, fyn * (Y[:, 1] / Yz) + cyn
    qmargin = torch.minimum(torch.minimum(qx, W - 1 - qx), torch.minimum(qy, H - 1 - qy))
    q_raw = torch.stack([qx, qy], -1).detach()
    ok = ok & (qmargin >= 0)
    qx, qy = _safe(ok, qx, 0.0), _safe(ok, qy, 0.0)
    Dn_raw = bilinear(depth_n.detach(), qx.detach(), qy.detach())
    taps_le0 = _taps_le0(depth_n.detach(), qx.detach(), qy.detach())
    ok_q = ok
    Dn = bilinear(depth_nf, qx, qy)
    ok = ok & (Dn_raw > 0) & torch.isfinite(Dn_raw)
    Dn = _safe(ok, Dn)
    un = torch.stack([(qx - cxn) / fxn, (qy - cyn) / fyn, torch.ones_like(qx)], -1)
    Xp = (Dn[:, None] * un - t) @ R
    ok_dn = ok
    ok = ok & (Xp[:, 2] > MIN_Z)
    Xz = _safe(ok, Xp[:, 2])
    ex, ey = fxr * (Xp[:, 0] / Xz) + cxr - xs, fyr * (Xp[:, 1] / Xz) + cyr - ys
    s2 = ex * ex + ey * ey
    phi = torch.where(s2 > 0, torch.sqrt(_safe(s2 > 0, s2)), torch.zeros_like(s2))
    pre_geo = ok
    geo = ok & (phi < tau)
    w = torch.exp(-phi).detach() if w is None else w
    geo_c = torch.where(geo, w * phi, torch.zeros_like(phi))

    # photometric, on geo-valid pixels only
    idx = geo.nonzero().squeeze(1)
    n_w = normal_r.reshape(3, -1).T[idx]
    n_c = F.normalize(n_w @ Rr.T, dim=-1)
    nlen = (n_w @ Rr.T).detach().norm(dim=-1)
    Xg = X[idx]
    d = (n_c * Xg).sum(-1)
    pok = d.abs() > MIN_Z
    m = n_c / _safe(pok, d)[:, None]
    M = R[None] + t[None, :, None] * m[:, None, :]
    Kn = torch.tensor([[fxn, 0, cxn], [0, fyn, cyn], [0, 0, 1]], dtype=dtype, device=dev)
    Kri = torch.tensor([[1 / fxr, 0, -cxr / fxr], [0, 1 / fyr, -cyr / fyr], [0, 0, 1]], dtype=dtype, device=dev)
    Hm = Kn @ M @ Kri
    gpad = F.pad(gray_r, (3, 3, 3, 3))
    px, py = xs[idx], ys[idx]
    ixl, iyl = px.long(), py.long()
    Sa = Sb = Saa = Sbb = Sab = 0
    hz_min = torch.full_like(d, float("inf"))
    hz_border = torch.full_like(d, float("inf"))      # |h.z - MIN_Z| over the magnitude of h.z's terms
    tap_grid = torch.full_like(d, float("inf"))       # the warped taps' least margin to a grid line (see _grid)
    for ky in range(-3, 4):
        for kx in range(-3, 4):
            P = torch.stack([px + kx, py + ky, torch.ones_like(px)], -1)
            h = (Hm @ P[:, :, None]).squeeze(-1)
            hz_min = torch.minimum(hz_min, h[:, 2].detach())
            hz_border = torch.minimum(hz_border, ((h[:, 2] - MIN_Z).abs() / (Hm[:, 2].abs() * P.abs()).sum(-1)).detach())
            hok = h[:, 2] > MIN_Z
            pok = pok & hok
            hz = _safe(hok, h[:, 2])
            b = bilinear(gray_n, h[:, 0] / hz, h[:, 1] / hz)
            tap_grid = torch.minimum(tap_grid, torch.minimum(_grid(h[:, 0] / hz, W), _grid(h[:, 1] / hz, H)))
            a = gpad[iyl + 3 + ky, ixl + 3 + kx]
            Sa, Sb, Saa, Sbb, Sab = Sa + a, Sb + b, Saa + a * a, Sbb + b * b, Sab + a * b
    ma, mb = Sa / 49, Sb / 49
    cov = Sab / 49 - ma * mb
    va, vb = Saa / 49 - ma * ma, Sbb / 49 - mb * mb
    ncc = cov / torch.sqrt(va * vb + NCC_EPS)
    c = torch.clamp(1 - ncc, 0, 2)
    photo = pok & (c < MAX_COST)
    photo_c = torch.zeros_like(phi).index_put((idx,), torch.where(photo, w[idx] * c, torch.zeros_like(c)))
    photo_full = torch.zeros_like(geo).index_put((idx,), photo)
    # the margins of every decision, for telling fp32 / fp64 disagreements apart (inf where it does not apply)
    inf = torch.full_like(phi, float("inf")).detach()
    c_full = inf.clone().index_put((idx,), c.detach())
    ncc_m = inf.clone().index_put((idx,), (1 - ncc).detach().abs())
    d_full = inf.clone().index_put((idx,), d.detach().abs())
    hz_full = inf.clone().index_put((idx,), hz_min)
    # the other decision quantities, NaN where the pixel never reaches them
    nan = torch.full_like(phi, float("nan")).detach()
    on_geo = lambda v: nan.clone().index_put((idx,), v.detach())
    reached = lambda mask, v: torch.where(mask, v.detach(), nan)
    return {"geo_c": geo_c, "photo_c": photo_c, "geo": geo, "photo": photo_full, "phi": phi.detach(),
            "pre_geo": pre_geo, "w": w, "q": torch.stack([qx, qy], -1).detach(), "qmargin": qmargin.detach(),
            "Dn": Dn.detach(), "c": c_full, "ncc_margin": ncc_m, "d": d_full, "hz": hz_full,
            "q_raw": q_raw, "D": D_raw.detach(), "Y2": reached(D > 0, Y[:, 2]), "Dn_raw": reached(ok_q, Dn_raw),
            "taps_le0": torch.where(ok_q, taps_le0, torch.zeros_like(taps_le0)), "P2": reached(ok_dn, Xp[:, 2]),
            "d_signed": on_geo(d), "va": on_geo(va), "vb": on_geo(vb), "ncc": on_geo(ncc), "nlen": on_geo(nlen),
            "hz_border": on_geo(hz_border),
            "q_grid": torch.minimum(_grid(q_raw[:, 0], W), _grid(q_raw[:, 1], H)), "tap_grid": on_geo(tap_grid)}


def consistency(depth, normal, gray, cams, pairs, tau=1.0, counts=None, info=False, weights=None):
    """(geo [B], photo [B]) of depth [V,1,H,W], normal [V,3,H,W], gray [V,1,H,W] (one dtype and device), `cams` V Cam
    and `pairs` B (r, n).  `counts` [B,2] replaces the valid-pixel counts in the denominators (the tests pass the
    kernel's, so that a pixel on a decision boundary changes no other pixel's gradient); `weights` (B per-pixel
    tensors) replaces w = exp(-phi), which carries no gradient, e.g. to hold it fixed under finite differences.  With
    info=True also the per-pair per-pixel dicts of _pair."""
    dtype = depth.dtype
    geos, photos, infos = [], [], []
    for b, (r, n) in enumerate(pairs):
        e = _pair(depth[r, 0], depth[n, 0], normal[r], gray[r, 0], gray[n, 0], cams[r], cams[n], tau, dtype,
                  None if weights is None else weights[b])
        cg, cp = e["geo"].sum(), e["photo"].sum()
        if counts is not None:
            cg, cp = int(counts[b][0]), int(counts[b][1])
        geos.append(e["geo_c"].sum() / max(int(cg), 1))
        photos.append(e["photo_c"].sum() / max(int(cp), 1))
        infos.append(e)
    out = torch.stack(geos), torch.stack(photos)
    return (*out, infos) if info else out


def borderline(e, tau, W, H, delta=5e-4):
    """Pixels of one pair (dict of _pair, fp64) whose validity an fp32 evaluation may decide differently: a decision
    quantity within `delta` of its threshold.  Returns (geo-borderline, photo-borderline) boolean [H*W]."""
    pre = e["pre_geo"]
    g = (e["qmargin"].abs() < delta) | (pre & ((e["phi"] - tau).abs() < delta)) | (pre & (e["Dn"].abs() < delta))
    p = e["geo"] & (((e["c"] - MAX_COST).abs() < delta) | (e["d"] < 1e-5) | (e["hz"] < 1e-5))
    return g, p


def borderline_edges(e, tau, W, H, delta=5e-4):
    """borderline() for adversarial maps: the same phi, q and c margins, and the decisions whose fp32 evaluation is
    ill-conditioned rather than merely close, each measured against the scale of its own terms: Y.z and X'.z near
    MIN_Z against the depth (the reprojection divides by them), D' near 0 against the depth (a tap next to a hole),
    |d| near MIN_Z against the depth, and h.z near MIN_Z against its terms."""
    pre = e["pre_geo"]
    D = torch.where(e["D"] > 0, e["D"], torch.zeros_like(e["D"]))
    near = lambda v, at, bound: torch.nan_to_num((v - at).abs(), nan=float("inf")) < bound
    q = e["q_raw"]
    margin = e["qmargin"].abs()
    for axis, extent in ((0, W), (1, H)):      # a one-pixel axis has both bounds at 0: exactly 0 there is decided
        if extent == 1:
            other = q[:, 1 - axis]
            rest = torch.minimum(other, (H if axis == 0 else W) - 1 - other).abs()
            margin = torch.where(q[:, axis] == 0, rest if (H if axis == 0 else W) > 1 else torch.full_like(rest, 1.0),
                                 margin)
    g = (margin < delta) | (pre & ((e["phi"] - tau).abs() < delta)) | near(e["Y2"], MIN_Z, 1e-3 * D) \
        | near(e["P2"], MIN_Z, 1e-3 * e["Dn_raw"].abs()) | near(e["Dn_raw"], 0.0, delta * D)
    nc = (e["nlen"] / 1e-12).clamp(max=1.0)                    # |n_c|
    p = e["geo"] & (((e["c"] - MAX_COST).abs() < delta) | near(e["d"], MIN_Z, 1e-6 * D * nc)
                    | near(e["hz_border"], 0.0, 1e-5))
    return g, p


# ---- scenes ------------------------------------------------------------------------------------------------------


def look_at(C, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """Row-vector world -> camera matrix [4,4] (float64) of a camera at C looking at target, x right, y down."""
    C = torch.tensor(C, dtype=torch.float64)
    fwd = torch.tensor(target, dtype=torch.float64) - C
    fwd = fwd / fwd.norm()
    right = torch.linalg.cross(fwd, torch.tensor(up, dtype=torch.float64))
    right = right / right.norm()
    down = torch.linalg.cross(fwd, right)
    Rc = torch.stack([right, down, fwd], 1)
    V = torch.eye(4, dtype=torch.float64)
    V[:3, :3] = Rc.T
    V[:3, 3] = -Rc.T @ C
    return V.T.contiguous()


def ring_cams(V, W, H, fovx=0.7, radius=4.0, spread_deg=6.0, elevation_deg=35.0):
    """V cameras a few degrees apart on a ring, looking at the origin (float32 view matrices)."""
    tx = math.tan(fovx / 2)
    ty = tx * H / W
    cams = []
    for v in range(V):
        az = math.radians(spread_deg * (v - (V - 1) / 2))
        el = math.radians(elevation_deg + 2.0 * (v % 2))
        C = (radius * math.cos(el) * math.cos(az), radius * math.cos(el) * math.sin(az), radius * math.sin(el))
        cams.append(Cam(look_at(C).float(), tx, ty, W / 2.0 + 0.37 * v, H / 2.0 - 0.21 * v))
    return cams


def _smooth(g, V, C, H, W, cell):
    """Smooth random fields [V,C,H,W] in float64: bicubic upsampling of coarse noise with one cell per `cell` px."""
    h, w = max(H // cell, 2) + 3, max(W // cell, 2) + 3
    z = torch.randn(V * C, 1, h, w, generator=g, dtype=torch.float64)
    return F.interpolate(z, size=(H, W), mode="bicubic", align_corners=True).reshape(V, C, H, W)


def plane_depth(cam, W, H, n_p, offset=0.0):
    """Camera z of the plane n_p . X = offset along every pixel ray (float64 [H,W]), and the world points [H,W,3]."""
    V = cam.viewmatrix.double()
    Rr, tr = V[:3, :3].T, V[3, :3]
    fx, fy = W / (2 * cam.tanfovx), H / (2 * cam.tanfovy)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    u = torch.stack([(xs - cam.cx) / fx, (ys - cam.cy) / fy, torch.ones_like(xs)], -1)
    n = torch.tensor(n_p, dtype=torch.float64)
    nc = Rr @ n                                   # plane normal in the camera frame; camera-frame plane nc . Xc = k
    k = offset + n @ (Rr.T @ tr)
    D = k / (u @ nc)
    Xc = D[..., None] * u
    Xw = (Xc - tr) @ Rr
    return D, Xw


def plane_scene(W, H, V=2, n_p=(0.15, -0.1, 1.0), period_px=14.0):
    """V cameras viewing the tilted plane n_p . X = 0 with a smooth sinusoidal texture whose period is about
    `period_px` pixels: exact depth, world normal and grey maps (float64, CPU) and the cameras."""
    cams = ring_cams(V, W, H)
    f = 2 * math.pi * (W / (2 * cams[0].tanfovx)) / (4.0 * period_px)      # world frequency at the ring's distance
    n = torch.tensor(n_p, dtype=torch.float64)
    n = n / n.norm()
    e1 = torch.linalg.cross(n, torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64))
    e1 = e1 / e1.norm()
    e2 = torch.linalg.cross(n, e1)
    depth, gray = [], []
    for cam in cams:
        D, Xw = plane_depth(cam, W, H, n.tolist())
        s1, s2 = Xw @ e1, Xw @ e2
        depth.append(D)
        gray.append(0.5 + 0.2 * torch.sin(f * s1) + 0.2 * torch.sin(0.8 * f * s2 + 0.5))
    depth = torch.stack(depth)[:, None]
    gray = torch.stack(gray)[:, None]
    normal = n.reshape(1, 3, 1, 1).expand(V, 3, H, W).contiguous()
    return depth, normal, gray, cams


def random_scene(W, H, V, seed=0):
    """Smooth random maps over the plane scene: the plane's depth with a smooth relative perturbation of a few percent
    (reprojection errors from 0 to several pixels), smooth random normals around the plane's, and a smooth random
    texture with features every ~8 pixels.  float64, CPU."""
    g = torch.Generator().manual_seed(seed)
    depth, normal, gray, cams = plane_scene(W, H, V)
    scale = 4.0 / W                      # reprojection errors of about 0.6 |noise| px
    depth = depth * (1 + scale * _smooth(g, V, 1, H, W, 24))
    normal = normal + 0.3 * _smooth(g, V, 3, H, W, 16)
    gray = (gray + 0.15 * _smooth(g, V, 1, H, W, 6)).clamp(0, 1)
    return depth, normal, gray, cams
