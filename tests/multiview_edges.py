"""Adversarial scenes for the multi-view consistency losses: silhouettes and holes, points behind the neighbour,
degenerate planes and normals, flat and inverted texture, tiny images, unequal intrinsics, 64 pairs and scaled scenes.

Each builder returns (depth, normal, gray, cams) in float64 on the CPU, like multiview_oracle.random_scene.  SCENES
maps a name to (builder, pairs, coverage): coverage(infos, maps) gives, for every branch the scene exists for, the
number of pixels that take it (from the fp64 oracle's per-pixel dicts) and the least number the scene must keep, so a
later edit to a scene cannot silently stop testing its branch."""
import math

import torch

import multiview_oracle as mo

PLANE = (0.15, -0.1, 1.0)
TINY_SIZES = [(1, 1), (1, 17), (5, 3), (7, 7), (15, 16), (17, 15), (33, 1), (4096, 8)]
SCALES = (1e-3, 1.0, 1e3)


def _unit(v):
    v = torch.tensor(v, dtype=torch.float64)
    return v / v.norm()


def textured_plane(cams, W, H, seed, n_p=PLANE, offset=0.0, noise=True):
    """Depth, world normal and grey maps of the textured plane n_p . X = offset seen by `cams` (float64 [V,C,H,W]).
    The texture is a function of the world point, so the views agree; with noise, smooth perturbations of a few
    percent of depth, 0.3 of normal and 0.15 of grey are added as in random_scene."""
    g = torch.Generator().manual_seed(seed)
    V = len(cams)
    n = _unit(n_p)
    e1 = torch.linalg.cross(n, torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64))
    e1 = e1 / e1.norm()
    e2 = torch.linalg.cross(n, e1)
    f = 2 * math.pi * (max(W, 64) / (2 * cams[0].tanfovx)) / (4.0 * 14.0)
    depth, gray, world = [], [], []
    for cam in cams:
        D, Xw = mo.plane_depth(cam, W, H, n.tolist(), offset)
        s1, s2 = Xw @ e1, Xw @ e2
        depth.append(D)
        world.append(Xw)
        gray.append(0.5 + 0.2 * torch.sin(f * s1) + 0.2 * torch.sin(0.8 * f * s2 + 0.5))
    depth, gray = torch.stack(depth)[:, None], torch.stack(gray)[:, None]
    normal = n.reshape(1, 3, 1, 1).expand(V, 3, H, W).contiguous()
    if noise:
        depth = depth * (1 + 4.0 / max(W, 32) * mo._smooth(g, V, 1, H, W, 24))
        normal = normal + 0.3 * mo._smooth(g, V, 3, H, W, 16)
        gray = (gray + 0.15 * mo._smooth(g, V, 1, H, W, 6)).clamp(0, 1)
    return depth, normal, gray, torch.stack(world)


def _stripes(W, H, k, width=8):
    """[H,W] stripe class of every pixel: (x // width) % k."""
    return (torch.arange(W) // width % k).expand(H, W)


def _rays(cam, W, H):
    fx, fy = W / (2 * cam.tanfovx), H / (2 * cam.tanfovy)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    return torch.stack([(xs - cam.cx) / fx, (ys - cam.cy) / fy, torch.ones_like(xs)], -1)


def _to_world(cam, n_c):
    """World normals [3,H,W] of camera-frame normals [H,W,3] (n_c = R_r n_w)."""
    Rr = cam.viewmatrix.double()[:3, :3].T
    return (n_c @ Rr).permute(2, 0, 1)


# ---- the scenes -------------------------------------------------------------------------------------------------


def silhouette(W=64, H=48, seed=1):
    """A textured disc 1.2 in front of the background plane (silhouettes with several pixels of parallax between the
    views, so some reprojections land on the other surface), and scattered holes in both views: 0, negative, +inf and
    -inf depths, so that bilinear taps straddle them."""
    cams = mo.ring_cams(2, W, H)
    depth, normal, gray, _ = textured_plane(cams, W, H, seed)
    fd, fn, fg, fw = textured_plane(cams, W, H, seed + 1, offset=1.2)
    centre = 1.2 * _unit(PLANE)
    disc = ((fw - centre).norm(dim=-1) < 0.7)[:, None] & (fd > 0)
    depth = torch.where(disc, fd, depth)
    normal = torch.where(disc, fn, normal)
    gray = torch.where(disc, 1 - fg, gray)
    g = torch.Generator().manual_seed(seed)
    r = torch.rand(depth.shape, generator=g, dtype=torch.float64)
    depth = torch.where(r < 0.04, torch.zeros_like(depth), depth)
    depth = torch.where((r >= 0.04) & (r < 0.05), -depth, depth)
    depth = torch.where((r >= 0.05) & (r < 0.055), torch.full_like(depth, math.inf), depth)
    depth = torch.where((r >= 0.055) & (r < 0.06), torch.full_like(depth, -math.inf), depth)
    return depth, normal, gray, cams


def behind(W=64, H=48, seed=2):
    """View 0 on the ring; views 1 and 2 a wide-angle camera standing on the plane and looking up towards view 0, so
    part of view 0's points lie behind it and part reproject outside its image.  View 2 has the same camera with every
    depth 50: the back-projection of pair (0, 2) lands behind view 0 (X'.z <= MIN_Z)."""
    ring = mo.ring_cams(1, W, H)[0]
    C0 = -(ring.viewmatrix.double()[3, :3] @ ring.viewmatrix.double()[:3, :3].T)
    C1 = (-0.6, 0.1, 0.35)
    up = mo.Cam(mo.look_at(C1, target=tuple(C0.tolist())).float(), 2.0, 1.5, W / 2 + 3.3, H / 2 - 1.7)
    cams = [ring, up, mo.Cam(up.viewmatrix.clone(), up.tanfovx, up.tanfovy, up.cx, up.cy)]
    depth, normal, gray, _ = textured_plane(cams, W, H, seed)
    depth[2] = 50.0
    return depth, normal, gray, cams


def degenerate(W=64, H=48, seed=3, scale_normals=True):
    """View 0's normals in stripes: regular; almost perpendicular to the pixel ray (n_c . u / |u| = s with
    |s| log-uniform in [1e-9, 1e-1], both signs: |d| around MIN_Z and plane horizons inside the 7x7 patch); pointing
    away; exactly zero; and of length 1e-13 and 1e-20 (below F.normalize's eps)."""
    cams = mo.ring_cams(2, W, H)
    depth, normal, gray, _ = textured_plane(cams, W, H, seed)
    g = torch.Generator().manual_seed(seed)
    cls = _stripes(W, H, 6)
    u = _rays(cams[0], W, H)
    uh = u / u.norm(dim=-1, keepdim=True)
    a = torch.randn(H, W, 3, generator=g, dtype=torch.float64)
    e = torch.linalg.cross(uh, a)
    e = e / e.norm(dim=-1, keepdim=True)
    s = 10 ** (-9 + 8 * torch.rand(H, W, 1, generator=g, dtype=torch.float64))
    s = s * torch.where(torch.rand(H, W, 1, generator=g) < 0.5, -1.0, 1.0).double()
    perp = _to_world(cams[0], (e + s * uh) / (1 + s * s).sqrt())
    n0 = normal[0]
    n0 = torch.where(cls == 1, perp, n0)
    n0 = torch.where(cls == 2, -n0, n0)
    n0 = torch.where(cls == 3, torch.zeros_like(n0), n0)
    if scale_normals:
        unit = n0 / n0.norm(dim=0, keepdim=True).clamp_min(1e-300)
        n0 = torch.where(cls == 4, 1e-13 * unit, n0)
        n0 = torch.where(cls == 5, 1e-20 * unit, n0)
    normal = normal.clone()
    normal[0] = n0
    return depth, normal, gray, cams


def flat(W=64, H=48, seed=4):
    """Flat and hostile texture.  View 0 in stripes: constant 0.5 (var a = 0), a fortieth of the contrast (var a var b
    below the 1e-8 floor), saturated at 0 and 1, regular; view 1 constant 0.5 in its right third (var b = 0); view 2 is view 1
    inverted (NCC near -1, c towards its clamp at 2, which population moments
    cannot pass)."""
    cams = mo.ring_cams(3, W, H)
    depth, normal, gray, _ = textured_plane(cams, W, H, seed)
    cls = _stripes(W, H, 4)
    low = 0.5 + 0.025 * (gray - 0.5)
    sat = (3 * (gray - 0.5) + 0.5).clamp(0, 1)
    g0 = gray[0, 0]
    g0 = torch.where(cls == 0, torch.full_like(g0, 0.5), g0)
    g0 = torch.where(cls == 1, low[0, 0], g0)
    g0 = torch.where(cls == 2, sat[0, 0], g0)
    gray = gray.clone()
    gray[0, 0] = g0
    gray[1, 0] = torch.where(cls == 1, low[1, 0], torch.where(cls == 2, sat[1, 0], gray[1, 0]))
    gray[1, 0, :, 2 * W // 3:] = 0.5
    gray[2] = 1 - gray[1]
    return depth, normal, gray, cams


def intrinsics(W=64, H=48, seed=5):
    """fx != fy in every view, principal points off centre, view 2's outside the image, and every pair's reference
    and neighbour intrinsics different."""
    ring = mo.ring_cams(3, W, H)
    spec = [(0.40, 0.40, 30.3, 20.9), (0.33, 0.21, 37.0, 27.5), (0.52, 0.45, -6.0, 50.5)]
    cams = [mo.Cam(c.viewmatrix, tx, ty, cx, cy) for c, (tx, ty, cx, cy) in zip(ring, spec)]
    depth, normal, gray, _ = textured_plane(cams, W, H, seed)
    return depth, normal, gray, cams


def tiny(W, H, seed=6):
    """The textured plane at an image smaller than the 7x7 patch or the 16x16 tile, or one pixel wide or high.  A valid
    pixel of a one-pixel axis reprojects exactly onto 0, so those images get axis-aligned cameras with the principal
    point at 0, translated along the other axis (along the optical axis for 1x1): the reprojection's coordinate on
    the one-pixel axis is then exactly 0 in fp32 as in fp64, and the perturbed depth keeps phi well away from 0."""
    if W > 1 and H > 1:
        cams = mo.ring_cams(2, W, H)
        depth, normal, gray, _ = textured_plane(cams, W, H, seed + W + 7 * H)
        return depth, normal, gray, cams
    shift = (0.0, 0.0, 0.3) if W == H == 1 else ((0.0, 0.25, 0.0) if W == 1 else (0.25, 0.0, 0.0))
    cams = []
    for C in ((0.0, 0.0, 0.0), shift):
        vm = torch.eye(4, dtype=torch.float64)
        vm[3, :3] = -torch.tensor(C, dtype=torch.float64)
        cams.append(mo.Cam(vm.float(), 0.5, 0.5, 0.0, 0.0))
    depth, normal, gray, _ = textured_plane(cams, W, H, seed + W + 7 * H, n_p=(0.2, -0.3, 1.0), offset=4.0)
    return depth, normal, gray, cams


def many(W=32, H=24, seed=7):
    """Nine views on the ring; view 8 has no depth at all, so its pairs count no pixel."""
    cams = mo.ring_cams(9, W, H, spread_deg=3.0)
    depth, normal, gray, _ = textured_plane(cams, W, H, seed)
    depth[8] = 0.0
    return depth, normal, gray, cams


def many_pairs(seed=7):
    """64 pairs: (v, v) for views 0-2 and 8 (the others keep pixels that no (v, v) pair puts on a grid line, so the
    per-pixel checks compare them), a pair repeated four times, neighbour 4 shared by all references, pairs of the
    empty view 8 as reference, and seeded random pairs to fill."""
    pairs = [(v, v) for v in (0, 1, 2, 8)] + [(0, 1)] * 4 + [(v, 4) for v in range(9) if v != 4] + [(8, v) for v in (0, 3, 7)]
    g = torch.Generator().manual_seed(seed)
    while len(pairs) < 64:
        r, n = torch.randint(0, 8, (2,), generator=g).tolist()
        pairs.append((r, n))
    return pairs


def scaled(s, W=64, H=48, seed=8):
    """The degenerate scene's regular and tiny-normal stripes with depths and camera translations times s."""
    depth, normal, gray, cams = degenerate(W, H, seed)
    cls = _stripes(W, H, 6)
    keep = (cls == 0) | (cls >= 4)
    normal[0] = torch.where(keep, normal[0], normal[1])
    out = []
    for c in cams:
        vm = c.viewmatrix.double().clone()
        vm[3, :3] *= s
        out.append(mo.Cam(vm.float(), c.tanfovx, c.tanfovy, c.cx, c.cy))
    return depth * s, normal, gray, out


# ---- coverage ---------------------------------------------------------------------------------------------------


def _n(mask):
    return int(torch.as_tensor(mask).sum())


def _valid(e, key, cond):
    v = e[key]
    return cond(v) & ~torch.isnan(v)


def cov_silhouette(infos, maps):
    depth = maps[0]
    e = infos[0]
    return {"hole D = 0": (_n(depth == 0), 100), "D < 0": (_n((depth < 0) & torch.isfinite(depth)), 30),
            "D = +inf": (_n(depth == math.inf), 10), "D = -inf": (_n(depth == -math.inf), 10),
            "other surface (phi >= tau)": (sum(_n(x["pre_geo"] & (x["phi"] >= 1.0)) for x in infos), 40),
            "taps straddle D <= 0": (sum(_n(x["geo"] & (x["taps_le0"] > 0)) for x in infos), 40),
            "Dn <= 0 at q": (sum(_n(_valid(x, "Dn_raw", lambda v: v <= 0)) for x in infos), 10),
            "geo-valid": (_n(e["geo"]), 1000), "photo-valid": (_n(e["photo"]), 200)}


def cov_behind(infos, maps):
    a, b = infos[0], infos[1]
    return {"Y.z <= MIN_Z": (_n(_valid(a, "Y2", lambda v: v <= mo.MIN_Z)), 100),
            "q outside the image": (_n(_valid(a, "Y2", lambda v: v > mo.MIN_Z) & (a["qmargin"] < 0)), 100),
            "X'.z <= MIN_Z": (_n(_valid(b, "P2", lambda v: v <= mo.MIN_Z)), 100),
            "geo-valid (0, 1)": (_n(a["geo"]), 15), "geo-valid (1, 0)": (_n(infos[2]["geo"]), 15)}


def cov_degenerate(infos, maps):
    e = infos[0]
    d = e["d_signed"]
    nl = e["nlen"]
    horizon = e["geo"] & (e["hz"] <= mo.MIN_Z) & (e["d"] > mo.MIN_Z)
    return {"|d| <= MIN_Z, |n| = 1": (_n(e["geo"] & (e["d"] <= mo.MIN_Z) & (nl > 0.5)), 20),
            "MIN_Z < |d| < 1e-3": (_n(e["geo"] & (e["d"] > mo.MIN_Z) & (e["d"] < 1e-3)), 20),
            "d < 0 photo-valid": (_n(e["photo"] & (d < 0)), 50),
            "horizon in the patch": (_n(horizon), 30), "zero normal": (_n(e["geo"] & (nl == 0)), 100),
            "|n| < eps photo-valid": (_n(e["photo"] & (nl < 1e-12)), 30),
            "|n| = 1e-20": (_n(e["geo"] & (nl < 1e-19) & (nl > 0)), 50),
            "photo-valid": (_n(e["photo"]), 300)}


def cov_flat(infos, maps):
    a, inv = infos[0], infos[1]
    gray = maps[2]
    return {"var a = 0": (_n(a["geo"] & (a["va"] < 1e-14)), 100),
            "var b = 0": (_n(a["geo"] & (a["vb"] < 1e-14)), 50),
            "var a var b < 1e-8 photo-valid": (_n(a["photo"] & (a["va"] * a["vb"] < 1e-8)), 15),
            "grey 0 or 1 in view 0": (_n((gray[0] == 0) | (gray[0] == 1)), 100),
            "saturated photo-valid": (_n(a["photo"] & (_stripes(maps[0].shape[3], maps[0].shape[2], 4) == 2)
                                         .reshape(-1).to(a["photo"].device)), 50),
            "inverted: c > 1.5": (_n(inv["geo"] & (inv["ncc"] < -0.5)), 100),
            "photo-valid (0, 1)": (_n(a["photo"]), 300)}


def cov_intrinsics(infos, maps):
    cams = maps[3]
    W, H = maps[0].shape[3], maps[0].shape[2]
    out = {"fx != fy": (sum(W / c.tanfovx != H / c.tanfovy for c in cams), 3),
           "principal point outside": (sum(not (0 <= c.cx < W and 0 <= c.cy < H) for c in cams), 1)}
    for b, e in enumerate(infos):
        out[f"geo-valid pair {b}"] = (_n(e["geo"]), 200)
        out[f"photo-valid pair {b}"] = (_n(e["photo"]), 50)
    return out


TINY_LEAST = {(1, 1): (3, 3), (1, 17): (40, 40), (33, 1): (80, 80)}      # (geo, photo) over the pairs


def cov_tiny(infos, maps):
    H, W = maps[0].shape[2:]
    geo, photo = sum(_n(e["geo"]) for e in infos), sum(_n(e["photo"]) for e in infos)
    lg, lp = TINY_LEAST.get((W, H), (H * W // 2, H * W // 4))
    return {"geo-valid": (geo, lg), "photo-valid": (photo, lp)}


def cov_many(infos, maps):
    counts = [_n(e["geo"]) for e in infos]
    return {"pairs": (len(infos), 64), "empty pairs": (sum(c == 0 for c in counts), 5),
            "pairs with >= 300 pixels": (sum(c >= 300 for c in counts), 20)}


def cov_scaled(infos, maps):
    e = infos[0]
    return {"|n| < eps photo-valid": (_n(e["photo"] & (e["nlen"] < 1e-12)), 30), "geo-valid": (_n(e["geo"]), 1000)}


SCENES = {
    "silhouette": (silhouette, [(0, 1), (1, 0)], cov_silhouette),
    "behind": (behind, [(0, 1), (0, 2), (1, 0)], cov_behind),
    "degenerate": (degenerate, [(0, 1), (1, 0)], cov_degenerate),
    "flat": (flat, [(0, 1), (0, 2), (1, 0)], cov_flat),
    "intrinsics": (intrinsics, [(0, 1), (1, 2), (2, 0), (0, 2)], cov_intrinsics),
    "many": (many, many_pairs(), cov_many),
}
for _W, _H in TINY_SIZES:
    SCENES[f"tiny{_W}x{_H}"] = ((lambda W=_W, H=_H: tiny(W, H)), [(0, 1), (1, 0), (0, 0)], cov_tiny)
for _s in SCALES:
    SCENES[f"scale{_s:g}"] = ((lambda s=_s: scaled(s)), [(0, 1), (1, 0)], cov_scaled)
