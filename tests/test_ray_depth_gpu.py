"""The ray-depth rasterizer mode on the GPU: off is off, on changes only the depth-derived outputs, the depth against an
fp64 recomposite on the kernel's own lists, the geometry it is for (flat Gaussians on a tilted plane), the gradients
against fp64 autograd of the same map, and the mode's composition with the rasterizer's other modes."""
import math

import pytest
import torch

import raydepth64
from helpers import EDGE_CASES, _edge_scene
from relightable3dgaussian_b200 import _C_raster, synth
from relightable3dgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
NAMES = ("n_contrib", "color", "opacity", "depth", "feature", "normal", "xyz", "weights", "radii")
DEPTH_OUTPUTS = ("depth", "normal", "xyz")


def _bits_equal(a, b):
    return a.shape == b.shape and bool((a.contiguous().view(torch.int32) == b.contiguous().view(torch.int32)).all())


def _leaves(P, S, seed=0, recipe="shell-v1", boost=1.0):
    sc = synth.make_scene(P, recipe, seed, S)
    f = lambda t: t.to(DEV).float().contiguous().requires_grad_(True)         # noqa: E731
    feats = sc.features if sc.features is not None else torch.zeros(P, 0)
    return dict(means3D=f(sc.means3D), opacities=f(sc.opacities), shs=f(sc.shs), scales=f(sc.scales * boost),
                rotations=f(sc.rotations), features=f(feats))


def _settings(cam, W, H, bg=(0.1, 0.2, 0.3), cam_grad=False):
    t = lambda x: x.to(DEV).float().contiguous().requires_grad_(cam_grad)     # noqa: E731
    return R.GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                           torch.tensor(bg, device=DEV), 1.0, t(cam.viewmatrix), t(cam.projmatrix),
                                           3, t(cam.campos), False, True, True, False)


def _run(lv, rs, cots=None, det=False, surface_grads=False, means2d_grad=True, **kw):
    """Forward and (with `cots`) backward; returns (outputs dict, gradients dict)."""
    torch.use_deterministic_algorithms(det)
    try:
        P = lv["means3D"].shape[0]
        m2 = torch.zeros(P, 3, device=DEV, requires_grad=means2d_grad)
        out = R.GaussianRasterizer(rs, surface_grads=surface_grads, **kw)(
            means3D=lv["means3D"], means2D=m2, opacities=lv["opacities"], shs=lv["shs"], scales=lv["scales"],
            rotations=lv["rotations"], features=lv["features"])
        o = dict(zip(NAMES, out[1:]))
        g = {}
        if cots is not None:
            loss = sum((o[k] * c).sum() for k, c in cots.items())
            leaves = dict(lv, means2D=m2)
            if rs.viewmatrix.requires_grad:
                leaves["viewmatrix"] = rs.viewmatrix
            names = [k for k, v in leaves.items() if v.requires_grad]
            gs = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
            g = {k: v for k, v in zip(names, gs) if v is not None}
            if getattr(m2, "absgrad", None) is not None:
                g["absgrad"] = m2.absgrad
        torch.cuda.synchronize()
        return {k: v.detach() for k, v in o.items()}, g
    finally:
        torch.use_deterministic_algorithms(False)


def _cots(W, H, S, depth_only=False, scale=1.0, seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda c: torch.randn(c, H, W, device=DEV, generator=g) * scale       # noqa: E731
    if depth_only:
        return {"depth": r(1)}
    return {"color": r(3), "opacity": r(1), "depth": r(1), "feature": r(S)}


SCENES = [("shell-v1", 3000, 5, 1.0), ("shell-v1", 1500, 16, 2.5)]


@pytest.mark.parametrize("det", [False, True])
def test_mode_off_is_off(det):
    """ray_depth=False is the default call: every output and gradient bitwise (default mode: up to atomic order)."""
    W, H = 160, 120
    lv = _leaves(2000, 5)
    rs = _settings(synth.make_camera(2, W, H), W, H)
    cots = _cots(W, H, 5)
    o0, g0 = _run(lv, rs, cots, det=det)
    o1, g1 = _run(lv, rs, cots, det=det, ray_depth=False)
    for k in NAMES:
        if k != "weights" or det:
            assert _bits_equal(o0[k], o1[k]), k
    for k in g0:
        if det:
            assert _bits_equal(g0[k], g1[k]), k
        else:
            assert float((g0[k] - g1[k]).norm() / g0[k].norm().clamp_min(1e-30)) <= 1e-5, k


@pytest.mark.parametrize("recipe,P,S,boost", SCENES + [("cube-v1", 2000, 1, 1.0), ("shell-v1", 500, 0, 6.0)])
def test_mode_on_changes_only_the_depth_outputs(recipe, P, S, boost):
    W, H = 200, 136
    lv = _leaves(P, S, recipe=recipe, boost=boost)
    for view in (0, 3):
        rs = _settings(synth.make_camera(view, W, H), W, H)
        off, _ = _run(lv, rs, det=True)
        on, _ = _run(lv, rs, det=True, ray_depth=True)
        for k in NAMES:
            if k in DEPTH_OUTPUTS:
                assert torch.isfinite(on[k]).all(), k
            else:
                assert _bits_equal(on[k], off[k]), (recipe, view, k)
        assert not _bits_equal(on["depth"], off["depth"])


@pytest.mark.parametrize("name", EDGE_CASES)
def test_mode_on_changes_only_the_depth_outputs_on_the_edge_cases(name):
    """Every edge-case scene of the rasterizer suites (near plane, frustum clamp, needles, saturation, sort keys,
    thresholds, strips, precomputed covariances): forward outputs other than the depth ones are bitwise mode-off."""
    sc, cam, S = _edge_scene(name)
    W, H = cam.image_width, cam.image_height
    rs = _settings(cam, W, H)._replace(scale_modifier=float(sc.get("scale_modifier", 1.0)))
    d = lambda t: None if t is None else t.to(DEV).float().contiguous()       # noqa: E731
    P = sc["means3D"].shape[0]
    args = dict(means3D=d(sc["means3D"]), means2D=torch.zeros(P, 3, device=DEV), opacities=d(sc["opacities"]),
                shs=d(sc.get("shs")), colors_precomp=d(sc.get("colors_precomp")), scales=d(sc.get("scales")),
                rotations=d(sc.get("rotations")), cov3D_precomp=d(sc.get("cov3D_precomp")),
                features=d(sc.get("features")))
    outs = []
    torch.use_deterministic_algorithms(True)
    try:
        for rd in (False, True):
            outs.append(dict(zip(NAMES, R.GaussianRasterizer(rs, ray_depth=rd)(**args)[1:])))
    finally:
        torch.use_deterministic_algorithms(False)
    for k in NAMES:
        if k in DEPTH_OUTPUTS:
            assert torch.isfinite(outs[1][k]).all(), (name, k)
        else:
            assert _bits_equal(outs[1][k], outs[0][k]), (name, k)


def _lists(rs, lv, W, H):
    """The kernel's per-pixel lists: the tile's depth-sorted ids and n_contrib (mode-off buffers: the same lists)."""
    out = _C_raster.rasterize_gaussians(rs.bg, lv["means3D"].detach(), lv["features"].detach(), torch.Tensor([]),
                                        lv["opacities"].detach(), lv["scales"].detach(), lv["rotations"].detach(),
                                        1.0, torch.Tensor([]), rs.viewmatrix.detach(), rs.projmatrix.detach(),
                                        rs.tanfovx, rs.tanfovy, rs.cx, rs.cy, H, W, lv["shs"].detach(), 3,
                                        rs.campos.detach(), False, True, False)
    P = lv["means3D"].shape[0]
    geom, binning, img = out[10], out[11], out[12]
    pl = _C_raster.debug_intermediate("point_list", P, 0, W, H, geom, img, binning, out[0]).long().cpu()
    ranges = _C_raster.debug_intermediate("ranges", P, 0, W, H, geom, img, binning, out[0]).long().cpu()
    nc = out[1].cpu().reshape(-1)
    gx = (W + 15) // 16
    order = []
    for pix in range(H * W):
        t = (pix // W // 16) * gx + (pix % W) // 16
        order.append(pl[ranges[t, 0]:ranges[t, 1]])
    return order, nc


def _record64(lv, cam, W, H, ray_depth=True):
    """fp64 (mean2D px, conic, opacity, tz, plane) of every Gaussian (raydepth64 / proj64 closed forms)."""
    import aa_oracle
    import proj64
    c64 = proj64.Camera(cam.viewmatrix, cam.projmatrix, cam.campos, W, H, cam.tanfovx, cam.tanfovy)
    m = lv["means3D"].detach().double().cpu()
    sig = aa_oracle.cov3d_of(lv["scales"].detach().double().cpu(), lv["rotations"].detach().double().cpu())
    P = m.shape[0]
    mean2D, conic, tz, p = torch.zeros(P, 2, dtype=torch.float64), torch.zeros(P, 3, dtype=torch.float64), \
        torch.zeros(P, dtype=torch.float64), torch.zeros(P, 2, dtype=torch.float64)
    for i in range(P):
        a0, b, c0, t = proj64.cov2d(m[i], sig[i], c64)
        a, c = a0 + 0.3, c0 + 0.3
        det = a * c - b * b
        conic[i] = torch.stack([c / det, -b / det, a / det])
        tz[i] = t
        p[i] = raydepth64.plane(m[i], sig[i], c64, linearised=False)
        h = m[i] @ c64.P[:3, :] + c64.P[3, :]
        ndc = h[:2] / (h[3] + 1e-7)
        mean2D[i] = ((ndc + 1.0) * torch.tensor([W, H], dtype=torch.float64) - 1.0) * 0.5
    return mean2D, conic, lv["opacities"].detach().double().cpu().reshape(-1), tz, p


def test_depth_against_fp64_recomposite():
    """The plane depth image against an fp64 recomposite on the kernel's own lists and n_contrib.  Pixels where the
    mode-off depth already disagrees with the same recomposite (an alpha or stop decision that fp32 and fp64 take
    differently) are ambiguous and excluded, as raster64 excludes them."""
    W, H = 64, 48
    cam = synth.make_camera(1, W, H)
    lv = _leaves(400, 1, seed=4, boost=2.0)
    rs = _settings(cam, W, H)
    off, _ = _run(lv, rs)
    on, _ = _run(lv, rs, ray_depth=True)
    order, nc = _lists(rs, lv, W, H)
    rec = _record64(lv, cam, W, H)
    want_off = raydepth64.composite_depth(*rec, order, nc, W, H, ray_depth=False)
    want_on = raydepth64.composite_depth(*rec, order, nc, W, H, ray_depth=True)
    scale = float(want_off.abs().max())
    ok = (off["depth"][0].double().cpu() - want_off).abs() <= 1e-4 * scale
    assert float(ok.double().mean()) > 0.95
    err = ((on["depth"][0].double().cpu() - want_on).abs() / scale)[ok]
    assert float(err.max()) <= 1e-4, float(err.max())


def _tilted_plane(W, H, slope=0.5, z0=3.0, spacing=0.025, s=0.03, thickness=0.001):
    """Flat discs on the camera-frame plane z = z0 + slope x (axis camera: camera frame = world frame)."""
    xs = torch.arange(-0.9, 0.9 + 1e-9, spacing, dtype=torch.float64)
    ys = torch.arange(-0.7, 0.7 + 1e-9, spacing, dtype=torch.float64)
    X, Y = torch.meshgrid(xs, ys, indexing="ij")
    X, Y = X.reshape(-1), Y.reshape(-1)
    Z = z0 + slope * X
    phi = -math.atan(slope)                                        # rotate e_z onto the plane normal about y
    P = X.numel()
    rot = torch.tensor([math.cos(phi / 2), 0.0, math.sin(phi / 2), 0.0]).repeat(P, 1)
    f = lambda t: t.to(DEV).float().contiguous().requires_grad_(True)         # noqa: E731
    lv = dict(means3D=f(torch.stack([X, Y, Z], 1)), opacities=f(torch.full((P, 1), 0.95)),
              shs=f(torch.zeros(P, 16, 3)), scales=f(torch.tensor([s, s, thickness]).repeat(P, 1)),
              rotations=f(rot), features=f(torch.zeros(P, 1)))
    return lv


def test_tilted_plane_depth_and_pseudo_normal():
    """Flat Gaussians lying on a tilted plane with known depth and normal.

    Depth bound.  Along image x the plane's depth is Z(u) = z0 / (1 - slope u), u = (x + 0.5 - W/2) / f.  A Gaussian's
    plane depth is the first-order expansion of Z at its centre, up to (a) the second-order term 0.5 |Z''| delta^2 at
    the pixel's offset delta from the centre, (b) the screen filter's shrinkage of the slope by 0.3 / (sigma_px^2 + 0.3)
    (the dilated conic), |Z'| delta of it, and (c) the disc's thickness.  delta <= 3.5 sigma_px for a composited
    entry.  The blended depth / opacity is a weighted mean of such depths, so it obeys the same bound."""
    W, H = 256, 192
    cam = synth.make_axis_camera(W, H)
    slope, z0, s, thick = 0.5, 3.0, 0.03, 0.001
    lv = _tilted_plane(W, H, slope, z0, s=s, thickness=thick)
    rs = _settings(cam, W, H, bg=(0.0, 0.0, 0.0))
    f = W / (2 * cam.tanfovx)
    x = torch.arange(W, dtype=torch.float64) + 0.5 - W / 2
    y = torch.arange(H, dtype=torch.float64) + 0.5 - H / 2
    u = (x / f)[None, :].expand(H, W)
    Ztrue = z0 / (1 - slope * u)
    Xtrue = u * Ztrue
    umax = float(u.abs().max())
    zmin = z0 / (1 + slope * umax)
    sigma_px = s * f / (z0 / (1 - slope * umax))                    # the smallest screen sigma (farthest disc)
    delta = 3.5 * s * f / zmin                                      # the largest composited offset
    d1 = slope * z0 / ((1 - slope * umax) ** 2 * f)                 # max |dZ/dx| per pixel
    d2 = 2 * slope * slope * z0 / ((1 - slope * umax) ** 3 * f * f)  # max |d2Z/dx2|
    bound = 0.5 * d2 * delta ** 2 + 0.3 / (sigma_px ** 2 + 0.3) * d1 * delta + 3 * thick
    res = {}
    for mode in (False, True):
        o, _ = _run(lv, rs, ray_depth=mode)
        op = o["opacity"][0].double().cpu()
        d = o["depth"][0].double().cpu() / op.clamp_min(1e-7)
        interior = (op > 0.98) & (Xtrue.abs() < 0.75) & (y.abs()[:, None] / f * Ztrue < 0.55)
        interior[:2] = interior[-2:] = False
        interior[:, :2] = interior[:, -2:] = False
        n = o["normal"].double().cpu()
        n = n / n.norm(dim=0).clamp_min(1e-30)
        nt = torch.tensor([-slope, 0.0, 1.0], dtype=torch.float64)
        nt = nt / nt.norm()
        ang = torch.rad2deg(torch.acos((n * nt[:, None, None]).sum(0).abs().clamp(max=1.0)))
        res[mode] = (float((d - Ztrue).abs()[interior].max()), float(ang[interior].mean()), int(interior.sum()))
    print("tilted plane: bound", bound, "centre depth (max err, mean angle, px)", res[False],
          "ray depth", res[True])
    assert res[True][2] > 5000
    assert res[True][0] <= bound, (res, bound)
    assert res[False][0] > bound                                    # the centre depth's terraces do not meet it
    # first H100 run: mean angular error 0.0134 deg (ray depth) against 0.321 deg (centre depth), ratio 0.042
    assert res[True][1] <= 0.1 * res[False][1], res


# ---- gradients: fp64 autograd of the same map on the kernel's own lists -------------------------------------------
def _render64(lv, cam, W, H, order, nc, bg, ray_depth):
    """fp64 (color, opacity, depth, feature) of the Gaussians on the kernel's lists and n_contrib, differentiable in
    every leaf, with the projection backward's conventions (proj64): the frustum clamp (t0 a constant on clamped rows),
    the conic's +1e-7 linearised inverse and ndc = h / (w + 1e-7); the plane stage of raydepth64.  lv: means3D,
    opacities, (scales, rotations) or cov3D, colors, features, and off [P,3], a zero leaf whose gradient is the
    kernel's dL_dmeans2D (ndc x, ndc y added to the projected mean, tz to the composited depth).  Returns the images and
    the pixels whose fp32 alpha decisions are ambiguous (alpha within 1e-6 of 1/255 or of the 0.99 clamp)."""
    import aa_oracle
    import proj64
    V, Pm = cam["viewmatrix"], cam["projmatrix"]
    m, o, off = lv["means3D"], lv["opacities"].reshape(-1), lv["off"]
    sig = aa_oracle.cov3d_from_six(lv["cov3D"]) if "cov3D" in lv else aa_oracle.cov3d_of(lv["scales"], lv["rotations"])
    t = m @ V[:3, :3] + V[3, :3]
    tx, ty, z = t[:, 0], t[:, 1], t[:, 2]
    hx, hy = W / (2 * cam["tanfovx"]), H / (2 * cam["tanfovy"])
    t0x = proj64._clamp_t(tx, z, 1.3 * cam["tanfovx"])
    t0y = proj64._clamp_t(ty, z, 1.3 * cam["tanfovy"])
    zero = torch.zeros_like(z)
    J = torch.stack([hx / z, zero, -hx * t0x / (z * z), zero, hy / z, -hy * t0y / (z * z)], 1).view(-1, 2, 3)
    T = J @ V[:3, :3].T
    C = T @ sig @ T.transpose(1, 2)
    a, b, c = C[:, 0, 0] + 0.3, C[:, 0, 1], C[:, 1, 1] + 0.3
    det = a * c - b * b
    A, B, Cc = proj64._lin_div(c, det), proj64._lin_div(-b, det), proj64._lin_div(a, det)
    cvec = (T @ (sig @ V[:3, 2])[..., None])[..., 0]
    p = torch.stack([A * cvec[:, 0] + B * cvec[:, 1], B * cvec[:, 0] + Cc * cvec[:, 1]], 1)
    h = m @ Pm[:3, :] + Pm[3, :]
    ndc = h[:, :2] / (h[:, 3:4] + 1e-7) + off[:, :2]
    mean2D = ((ndc + 1.0) * torch.tensor([W, H], dtype=torch.float64, device=m.device) - 1.0) * 0.5
    ch = torch.cat([lv["colors"], lv["features"]], 1)
    L = max(1, max(int(x.numel()) for x in order))
    ids = torch.zeros(H * W, L, dtype=torch.long)
    valid = torch.zeros(H * W, L, dtype=torch.bool)
    for pix in range(H * W):
        k = int(nc[pix])
        ids[pix, :k] = order[pix][:k]
        valid[pix, :k] = True
    ids, valid = ids.to(m.device), valid.to(m.device)
    px = torch.arange(H * W, device=m.device)
    x, y = (px % W).double()[:, None], (px // W).double()[:, None]
    dx, dy = mean2D[ids, 0] - x, mean2D[ids, 1] - y
    power = -0.5 * (A[ids] * dx * dx + Cc[ids] * dy * dy) - B[ids] * dx * dy
    raw = o[ids] * torch.exp(power)
    amb = (valid & (((raw - 1.0 / 255.0).abs() < 1e-6) | ((raw - 0.99).abs() < 1e-6))).any(1).view(H, W)
    alpha = raw.clamp(max=0.99)
    keep = valid & (power <= 0) & (alpha >= 1.0 / 255.0)
    alpha = torch.where(keep, alpha, torch.zeros_like(alpha))
    Tr = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha[:, :-1]], 1), 1)
    w = alpha * Tr
    tz = z + off[:, 2]
    d = tz[ids] - p[ids, 0] * dx - p[ids, 1] * dy if ray_depth else tz[ids]
    Tf = Tr[:, -1] * (1 - alpha[:, -1])
    img = (w[..., None] * ch[ids]).sum(1)
    img = torch.cat([img[:, :3] + bg[None] * Tf[:, None], img[:, 3:]], 1).T.reshape(-1, H, W)
    return dict(color=img[:3], opacity=w.sum(1).view(1, H, W), depth=(w * d).sum(1).view(1, H, W),
                feature=img[3:]), amb


def _row_scene(kind, S=1):
    """(leaves [P,...] on the CPU, camera, W, H).  shell: scales / rotations; precomp: cov3D_precomp; clamp: a third of
    the Gaussians centred outside the frustum clamp (|x / z| > 1.3 tan fov) but wide enough to reach the image."""
    W, H = 64, 48
    g = torch.Generator().manual_seed(11)
    sc = synth.make_scene(300, "shell-v1", 7, S)
    cam = synth.make_camera(1, W, H)
    lv = dict(means3D=sc.means3D.clone(), opacities=sc.opacities.clone(), colors=torch.rand(300, 3, generator=g),
              features=sc.features.clone())
    if kind == "clamp":
        cam = synth.make_axis_camera(W, H)
        n = 300
        z = 2.0 + 2.0 * torch.rand(n, generator=g)
        r = torch.rand(n, 2, generator=g) * 2 - 1
        out = torch.rand(n, generator=g) < 0.33
        fx = torch.where(out, torch.sign(r[:, 0]) * (1.45 + 0.3 * torch.rand(n, generator=g)), r[:, 0])
        lv["means3D"] = torch.stack([fx * cam.tanfovx * z, r[:, 1] * cam.tanfovy * z, z], 1)
        s = torch.where(out, torch.full((n,), 0.35), 0.03 + 0.05 * torch.rand(n, generator=g))
        sc = sc._replace(scales=torch.stack([s, 0.6 * s, 0.3 * s], 1))
    import aa_oracle
    if kind == "precomp":
        c = aa_oracle.cov3d_of(sc.scales.double() * 2.0, sc.rotations.double())
        lv["cov3D"] = torch.stack([c[:, 0, 0], c[:, 0, 1], c[:, 0, 2], c[:, 1, 1], c[:, 1, 2], c[:, 2, 2]], 1).float()
    else:
        lv["scales"] = sc.scales * (1.0 if kind == "clamp" else 2.0)
        lv["rotations"] = sc.rotations.clone()
    return lv, cam, W, H


def _row_check(got, want, tau, what):
    """Per row: |g - g64| <= tau (max_row |g64| + 1e-6 max |g64|) (rows of a leaf, or the elements of a camera matrix)."""
    got, want = got.double().reshape(want.shape[0], -1), want.reshape(want.shape[0], -1)
    scale = want.abs().amax(1, keepdim=True) + 1e-6 * want.abs().max()
    r = (got - want).abs() / scale.clamp_min(1e-300)
    bad = (r > tau).any(1)
    assert not bool(bad.any()), (what, int(bad.sum()), float(r.max()))


@pytest.mark.parametrize("kind", ["shell", "clamp", "precomp"])
@pytest.mark.parametrize("ray_depth", [False, True])
@pytest.mark.parametrize("cot", ["unit-mixed", "unit-depth-only", "training-scale-mixed", "training-scale-depth-only"])
@pytest.mark.parametrize("det", [False, True])
def test_gradient_rows_against_fp64(kind, ray_depth, cot, det):
    """Every leaf gradient, per row, against fp64 autograd of the same projection (the projection backward's
    conventions: frustum clamp, linearised conic inverse) and compositing on the kernel's lists: means2D (the
    compositor's dL/dmean2D and dL/dtz slots, with d's -p dL/dtz), opacities, means3D, scales and rotations or
    cov3D_precomp (through dL/dconic and the plane's dL/dp slots), viewmatrix and projmatrix.  Pixels with an ambiguous
    fp32 alpha decision get no cotangent."""
    S = 1
    lv, cam, W, H = _row_scene(kind, S)
    P = lv["means3D"].shape[0]
    camt = {k: getattr(cam, k).to(DEV).float().contiguous().requires_grad_(True) for k in ("viewmatrix", "projmatrix")}
    rs = R.GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                         torch.tensor([0.1, 0.2, 0.3], device=DEV), 1.0, camt["viewmatrix"],
                                         camt["projmatrix"], 0, cam.campos.to(DEV), False, True, True, False)
    dev = {k: v.to(DEV).float().contiguous() for k, v in lv.items()}
    order, nc = _lists_of(rs, dev, W, H)
    lv64 = {k: v.to(DEV).double().requires_grad_(True) for k, v in lv.items()}
    lv64["off"] = torch.zeros(P, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    cam64 = dict(viewmatrix=cam.viewmatrix.to(DEV).double().requires_grad_(True),
                 projmatrix=cam.projmatrix.to(DEV).double().requires_grad_(True), tanfovx=cam.tanfovx,
                 tanfovy=cam.tanfovy)
    out64, amb = _render64(lv64, cam64, W, H, order, nc, rs.bg.double(), ray_depth)
    assert float(amb.double().mean()) < 0.05
    scale = 2.0 ** -21 if cot.startswith("training") else 1.0
    cots = {k: c * (~amb).float() for k, c in _cots(W, H, S, depth_only="depth-only" in cot, scale=scale).items()}
    loss = sum((out64[k] * c.double()).sum() for k, c in cots.items())
    leaf_names = ["means3D", "opacities"] + (["cov3D"] if "cov3D" in lv else ["scales", "rotations"])
    want = torch.autograd.grad(loss, [lv64[k] for k in leaf_names] + [lv64["off"], cam64["viewmatrix"],
                                                                       cam64["projmatrix"]])
    leaves = {k: dev[k].clone().requires_grad_(True) for k in leaf_names}
    m2 = torch.zeros(P, 3, device=DEV, requires_grad=True)
    torch.use_deterministic_algorithms(det)
    try:
        o = R.GaussianRasterizer(rs, ray_depth=ray_depth)(
            means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], colors_precomp=dev["colors"],
            scales=leaves.get("scales"), rotations=leaves.get("rotations"), cov3D_precomp=leaves.get("cov3D"),
            features=dev["features"])
        img = dict(color=o[2], opacity=o[3], depth=o[4], feature=o[5])
        loss32 = sum((img[k] * c).sum() for k, c in cots.items())
        got = torch.autograd.grad(loss32, [leaves[k] for k in leaf_names] + [m2, camt["viewmatrix"],
                                                                             camt["projmatrix"]])
    finally:
        torch.use_deterministic_algorithms(False)
    tau = 2e-3
    for k, g32, g64 in zip(leaf_names + ["means2D"], got, want):
        _row_check(g32, g64, tau, (kind, k))
    # camera matrices: the elements the projection reads (viewmatrix column 3 and projmatrix column 2 are never read)
    _row_check(got[-2].view(4, 4)[:, :3].reshape(1, -1), want[-2].view(4, 4)[:, :3].reshape(1, -1), tau,
               (kind, "viewmatrix"))
    _row_check(got[-1].view(4, 4)[:, [0, 1, 3]].reshape(1, -1), want[-1].view(4, 4)[:, [0, 1, 3]].reshape(1, -1), tau,
               (kind, "projmatrix"))


def _lists_of(rs, dev, W, H):
    """The kernel's per-pixel lists and n_contrib for the leaves `dev` (colors_precomp; default-mode buffers: the same
    lists as the mode's)."""
    empty = torch.Tensor([])
    out = _C_raster.rasterize_gaussians(rs.bg, dev["means3D"], dev["features"], dev["colors"], dev["opacities"],
                                        dev.get("scales", empty), dev.get("rotations", empty), 1.0,
                                        dev.get("cov3D", empty), rs.viewmatrix.detach(), rs.projmatrix.detach(),
                                        rs.tanfovx, rs.tanfovy, rs.cx, rs.cy, H, W, empty, 0, rs.campos, False, True,
                                        False, ray_depth=False)
    P = dev["means3D"].shape[0]
    pl = _C_raster.debug_intermediate("point_list", P, 0, W, H, out[10], out[12], out[11], out[0]).long().cpu()
    ranges = _C_raster.debug_intermediate("ranges", P, 0, W, H, out[10], out[12], out[11], out[0]).long().cpu()
    nc = out[1].cpu().reshape(-1)
    gx = (W + 15) // 16
    order = [pl[ranges[(pix // W // 16) * gx + (pix % W) // 16, 0]:ranges[(pix // W // 16) * gx + (pix % W) // 16, 1]]
             for pix in range(H * W)]
    return order, nc


@pytest.mark.parametrize("det", [True, False])
def test_zero_depth_cotangent_gives_the_mode_off_gradients(det):
    """With no depth cotangent (surface_grads off) the plane terms add exact zeros to the gradient rows: dL/dmean2D is
    bitwise the mode-off one in deterministic mode.  The leaf gradients agree to 1e-6 of their largest element, not
    bitwise: the mode's projection-backward instantiation contracts some of the shared chain's multiply-adds
    differently."""
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    rs = _settings(synth.make_camera(2, W, H), W, H, cam_grad=True)
    cots = _cots(W, H, S)
    cots["depth"] = torch.zeros_like(cots["depth"])
    _, g0 = _run(lv, rs, cots, det=det)
    _, g1 = _run(lv, rs, cots, det=det, ray_depth=True)
    for k in g0:
        if k == "means2D" and det:     # the compositor's rows: exact (== also equates the zeros' signs)
            assert bool((g0[k] == g1[k]).all()), k
        elif k == "means2D":           # float atomics: the order of the rows' additions only
            assert float((g0[k] - g1[k]).norm() / g0[k].norm()) <= 1e-5, k
        else:
            e = float((g0[k] - g1[k]).abs().max() / g0[k].abs().max())
            assert e <= (1e-6 if det else 2e-5), (k, e)          # default mode: float-atomic order on top


@pytest.mark.parametrize("S", [0, 1, 2, 4, 5, 9, 13, 16, 20, 21, 24, 25, 28, 29, 33])
def test_every_channel_group_runs_in_the_mode(S):
    W, H = 96, 64
    lv = _leaves(600, S, seed=S)
    rs = _settings(synth.make_camera(5, W, H), W, H)
    cots = _cots(W, H, S) if S <= 24 else None
    off, g_off = _run(lv, rs, cots, det=True)
    on, g_on = _run(lv, rs, cots, det=True, ray_depth=True)
    for k in NAMES:
        if k not in DEPTH_OUTPUTS:
            assert _bits_equal(on[k], off[k]), (S, k)
    for k in g_on:
        assert torch.isfinite(g_on[k]).all(), (S, k)
    if cots is not None:           # the appearance gradients do not involve the depth
        assert _bits_equal(g_on["features"], g_off["features"])
        assert _bits_equal(g_on["shs"], g_off["shs"])


def test_several_views_are_their_one_view_calls():
    W, H, S = 96, 64, 5
    lv = _leaves(1500, S)
    cams = [synth.make_camera(k, W, H) for k in (0, 3, 6)]
    settings = [_settings(c, W, H) for c in cams]
    torch.use_deterministic_algorithms(True)
    try:
        m2 = torch.zeros(3, 1500, 3, device=DEV, requires_grad=True)
        out = R.rasterize_views(lv["means3D"], m2, lv["opacities"], settings=settings, shs=lv["shs"],
                                scales=lv["scales"], rotations=lv["rotations"], features=lv["features"], ray_depth=True)
        gv = torch.autograd.grad(out[4].sum(), [lv["means3D"], m2])
    finally:
        torch.use_deterministic_algorithms(False)
    for v, rs in enumerate(settings):
        o, g = _run(lv, rs, {"depth": torch.ones(1, H, W, device=DEV)}, det=True, ray_depth=True)
        for k in NAMES:
            assert _bits_equal(out[1 + NAMES.index(k)][v], o[k]), (v, k)
        assert _bits_equal(gv[1][v], g["means2D"]), v


def test_deterministic_mode_is_reproducible():
    W, H, S = 160, 120, 5
    lv = _leaves(3000, S)
    rs = _settings(synth.make_camera(1, W, H), W, H, cam_grad=True)
    cots = _cots(W, H, S)
    _, a = _run(lv, rs, cots, det=True, ray_depth=True)
    _, b = _run(lv, rs, cots, det=True, ray_depth=True)
    for k in a:
        assert _bits_equal(a[k], b[k]), k


def test_frozen_geometry_gets_the_mode_off_appearance_gradients():
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    for k in ("means3D", "opacities", "scales", "rotations"):
        lv[k] = lv[k].detach()
    rs = _settings(synth.make_camera(2, W, H), W, H)
    cots = _cots(W, H, S)
    _, g0 = _run(lv, rs, cots, det=True, means2d_grad=False)
    _, g1 = _run(lv, rs, cots, det=True, means2d_grad=False, ray_depth=True)
    assert set(g0) == set(g1) == {"shs", "features"}
    for k in g0:
        assert _bits_equal(g0[k], g1[k]), k


def test_surface_gradients_in_the_mode():
    """surface_grads=True with the mode on: the pseudo-normal and surface-xyz cotangents run through the backward
    (finite gradients), deterministic mode reproducible."""
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    rs = _settings(synth.make_camera(2, W, H), W, H)
    g = torch.Generator(device=DEV).manual_seed(3)
    cots = {"color": torch.randn(3, H, W, device=DEV, generator=g), "opacity": torch.randn(1, H, W, device=DEV, generator=g),
            "normal": torch.randn(3, H, W, device=DEV, generator=g), "xyz": torch.randn(3, H, W, device=DEV, generator=g)}
    _, g1 = _run(lv, rs, cots, det=True, surface_grads=True, ray_depth=True)
    _, g2 = _run(lv, rs, cots, det=True, surface_grads=True, ray_depth=True)
    for k in ("means3D", "scales", "rotations", "means2D"):
        assert torch.isfinite(g1[k]).all() and _bits_equal(g1[k], g2[k]), k


@pytest.mark.parametrize("det", [False, True])
def test_absgrad_bounds_the_signed_gradient(det):
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    rs = _settings(synth.make_camera(2, W, H), W, H)
    cots = _cots(W, H, S)
    _, g = _run(lv, rs, cots, det=det, ray_depth=True, absgrad=True)
    _, g_noabs = _run(lv, rs, cots, det=True, ray_depth=True)
    assert bool((g["absgrad"] >= g["means2D"][:, :2].abs() * (1 - 1e-4) - 1e-30).all())
    if det:
        assert _bits_equal(g["means2D"], g_noabs["means2D"])


@pytest.mark.parametrize("variant", ["antialiasing", "filter_3d"])
def test_composes_with_antialiasing_and_the_3d_filter(variant):
    """Only the depth outputs change with the mode on top of either mode, and the gradients are finite."""
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    rs = _settings(synth.make_camera(2, W, H), W, H)
    kw = {"antialiasing": True}
    if variant == "filter_3d":
        kw = {}
    P = lv["means3D"].shape[0]
    f3d = torch.full((P,), 0.01, device=DEV)
    cots = _cots(W, H, S)

    def run(rd):
        torch.use_deterministic_algorithms(True)
        try:
            m2 = torch.zeros(P, 3, device=DEV, requires_grad=True)
            out = R.GaussianRasterizer(rs, ray_depth=rd, **kw)(
                means3D=lv["means3D"], means2D=m2, opacities=lv["opacities"], shs=lv["shs"], scales=lv["scales"],
                rotations=lv["rotations"], features=lv["features"], filter_3d=f3d if variant == "filter_3d" else None)
            o = dict(zip(NAMES, out[1:]))
            loss = sum((o[k] * c).sum() for k, c in cots.items())
            gr = torch.autograd.grad(loss, [lv["means3D"], lv["scales"]])
            return {k: v.detach() for k, v in o.items()}, gr
        finally:
            torch.use_deterministic_algorithms(False)
    off, _ = run(False)
    on, gr = run(True)
    for k in NAMES:
        if k not in DEPTH_OUTPUTS:
            assert _bits_equal(on[k], off[k]), k
    assert all(torch.isfinite(t).all() for t in gr)


def test_deferred_count_repair_reruns_the_forward_in_the_mode(monkeypatch):
    """A deferred-count forward whose binning buffer overflowed is re-run inside the backward with the mode on: the
    gradients equal those of a synchronous call."""
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    rs = _settings(synth.make_camera(2, W, H), W, H)
    cots = _cots(W, H, S, depth_only=True)
    _, want = _run(lv, rs, cots, det=True, ray_depth=True)
    R.set_deferred_count(True)
    orig = _C_raster.rasterize_gaussians
    calls = []

    def tiny_first(*a, **kw):
        calls.append(kw.get("ray_depth"))
        if len(calls) == 1 and kw.get("_defer"):
            kw["_min_capacity"] = 64                  # overflow on purpose: the count is learnt from the re-run
        return orig(*a, **kw)
    monkeypatch.setattr(R._C, "rasterize_gaussians", tiny_first)
    st = _C_raster._dev_state(DEV)
    seen = st["seen"]
    st["seen"] = 1 << 20                              # past the learning phase: the forward defers its count
    try:
        with pytest.warns(UserWarning, match="overflowed"):
            _, got = _run(lv, rs, cots, det=True, ray_depth=True)
    finally:
        st["seen"] = seen
        R.set_deferred_count(False)
    assert calls[0] is True and calls[-1] is True and len(calls) >= 2
    for k in want:
        assert _bits_equal(got[k], want[k]), k


class _ReferenceCallPattern(torch.autograd.Function):
    """The reference wrapper's calls (gaussian_renderer/r3dg_rasterization.py): positional arguments only, through the
    drop-in `r3dg_rasterization._C`, no keyword of this project."""

    @staticmethod
    def forward(ctx, C, rs, means3D, features, shs, opacities, scales, rotations):
        empty = torch.Tensor([])
        args = (rs.bg, means3D, features, empty, opacities, scales, rotations, rs.scale_modifier, empty, rs.viewmatrix,
                rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.cx, rs.cy, rs.image_height, rs.image_width, shs, rs.sh_degree,
                rs.campos, rs.prefiltered, rs.computer_pseudo_normal, rs.debug)
        out = C.rasterize_gaussians(*args)
        ctx.C, ctx.rs, ctx.num_rendered = C, rs, out[0]
        ctx.save_for_backward(means3D, features, shs, scales, rotations, out[9], *out[10:13])
        return out[1:10]

    @staticmethod
    def backward(ctx, g_nc, g_color, g_opacity, g_depth, g_feature, *rest):
        means3D, features, shs, scales, rotations, radii, geom, binning, img = ctx.saved_tensors
        rs, empty = ctx.rs, torch.Tensor([])
        args = (rs.bg, means3D, features, radii, empty, scales, rotations, rs.scale_modifier, empty, rs.viewmatrix,
                rs.projmatrix, rs.tanfovx, rs.tanfovy, g_color, g_opacity, g_depth, g_feature, shs, rs.sh_degree,
                rs.campos, geom, ctx.num_rendered, binning, img, rs.backward_geometry, rs.debug)
        g = ctx.C.rasterize_gaussians_backward(*args)
        return None, None, g[3], g[4], g[6], g[2], g[7], g[8]


@pytest.mark.parametrize("plug_in", [False, True])
def test_plug_in_line_reaches_the_reference_call_pattern(plug_in):
    """rasterizer.set_ray_depth(True) reaches a caller of the drop-in `_C` that passes no keyword (the reference's own
    wrapper): its forward and backward are then bitwise those of ray_depth=True, and without the line bitwise those of
    the default mode (deterministic mode)."""
    import importlib
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if os.path.join(root, "dropin") not in sys.path:
        sys.path.insert(0, os.path.join(root, "dropin"))
    C = importlib.import_module("r3dg_rasterization")._C
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    rs = _settings(synth.make_camera(2, W, H), W, H)
    cots = _cots(W, H, S)
    R.set_ray_depth(plug_in)
    torch.use_deterministic_algorithms(True)
    try:
        out = _ReferenceCallPattern.apply(C, rs, lv["means3D"], lv["features"], lv["shs"], lv["opacities"],
                                          lv["scales"], lv["rotations"])
        o = dict(color=out[1], opacity=out[2], depth=out[3], feature=out[4], normal=out[5])
        loss = sum((o[k] * c).sum() for k, c in cots.items())
        names = ("means3D", "opacities", "scales", "rotations", "features", "shs")
        g = dict(zip(names, torch.autograd.grad(loss, [lv[k] for k in names])))
    finally:
        torch.use_deterministic_algorithms(False)
        R.set_ray_depth(False)
    want_o, want_g = _run(lv, rs, cots, det=True, means2d_grad=False, ray_depth=plug_in)
    for k in ("color", "opacity", "depth", "feature", "normal"):
        assert _bits_equal(o[k].detach(), want_o[k]), k
    for k in names:
        assert _bits_equal(g[k], want_g[k]), k
    off_o, _ = _run(lv, rs, det=True, means2d_grad=False)
    assert _bits_equal(o["depth"].detach(), off_o["depth"]) != plug_in
