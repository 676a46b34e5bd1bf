"""Gradients of the rasterizer's pseudo-normal (output 6) and surface_xyz (output 7) with `surface_grads=True`.

The adjoint pass turns their cotangents into extra depth and opacity cotangents, which the backward compositor then
consumes unchanged.  Those combined planes are checked against torch autograd of an fp64 restatement of the forward
(tests/surface_oracle.py) evaluated on the forward's own fp32 images; the rest checks that the compositor consumes
exactly those planes, that the default path is untouched, several views, reproducibility, the deferred-count repair
and a two-way depth-normal consistency loss."""
import warnings

import pytest
import torch

from helpers import rel_l2
from relightable3dgaussian_b200 import _C_raster, _lib, synth
from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_views,
                                                   set_deferred_count)
from surface_oracle import ill_conditioned, surface_normal

pytestmark = pytest.mark.gpu

IMAGES = (2, 3, 4, 5)          # color, opacity, depth, feature
SURFACE = (6, 7)               # normal, surface_xyz


@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def make_leaves(P, S, seed=0):
    sc = synth.make_scene(P, seed=seed, S=S)
    leaves = dict(means3D=sc.means3D, opacities=sc.opacities, shs=sc.shs, scales=sc.scales, rotations=sc.rotations)
    if S > 0:
        leaves["features"] = sc.features
    return {k: v.cuda().contiguous().requires_grad_(True) for k, v in leaves.items()}


def cotangents(H, W, S, seed=5):
    """color, opacity, depth, feature, normal, surface_xyz"""
    g = torch.Generator().manual_seed(seed)
    return [t.cuda() for t in (torch.randn(3, H, W, generator=g), torch.randn(1, H, W, generator=g),
                               torch.randn(1, H, W, generator=g) * 0.1, torch.randn(S, H, W, generator=g),
                               torch.randn(3, H, W, generator=g), torch.randn(3, H, W, generator=g) * 0.1)]


def settings_of(cam, vm, pm, cp):
    return GaussianRasterizationSettings(cam.image_height, cam.image_width, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                         torch.tensor([0.1, 0.4, 0.7], device="cuda"), 1.0, vm, pm, 3, cp, False, True,
                                         True, False)


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def one_view(leaves, cam, cot, surface_grads, touch=True, plane_cot=None):
    """Every gradient of one view through the public API: {leaf..., means2D, viewmatrix, projmatrix, campos}, and the
    library's launch count of the backward.  `touch`: the loss includes the normal and surface_xyz terms.
    `plane_cot`: (opacity, depth) cotangents that replace the loss's own."""
    vm, pm, cp = (t.cuda().contiguous().requires_grad_(True) for t in (cam.viewmatrix, cam.projmatrix, cam.campos))
    P = leaves["means3D"].shape[0]
    m2d = torch.zeros(P, 3, device="cuda", requires_grad=True)
    kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
    out = GaussianRasterizer(settings_of(cam, vm, pm, cp), surface_grads=surface_grads)(
        leaves["means3D"], m2d, leaves["opacities"], **kw)
    cots = list(cot[:4])
    if plane_cot is not None:
        cots[1], cots[2] = plane_cot
    loss = sum((out[i] * c).sum() for i, c in zip(IMAGES, cots))
    if touch:
        loss = loss + sum((out[i] * c).sum() for i, c in zip(SURFACE, cot[4:]))
    names = list(leaves) + ["means2D", "viewmatrix", "projmatrix", "campos"]
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.r3dg_launch_count()
    gs = torch.autograd.grad(loss, list(leaves.values()) + [m2d, vm, pm, cp])
    torch.cuda.synchronize()
    return dict(zip(names, gs)), lib.r3dg_launch_count() - n0


def masked(cot, cam, opacity, depth):
    """The cotangents with the normal's cotangent zeroed on ill-conditioned pixels (surface_oracle.ill_conditioned):
    their exact derivative is ~1/|n| with |n| rounding noise, no yardstick for the kernel."""
    bad = ill_conditioned(opacity, depth, cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy)
    return list(cot[:4]) + [cot[4] * (~bad).float(), cot[5]], int(bad.sum())


def c_planes(leaves, cam, cot, V=1, cams=None):
    """Forward and surface backward through the host layer of the C ABI; returns the combined depth and opacity
    cotangent planes read from the workspace ([V,H,W] each), the camera partials summed in fp64 ([V,3,3]), the forward's
    opacity / depth images, the camera gradients and the cotangents used (masked()).  V > 1: `cams` and `cot` are per
    view."""
    d = {k: t.detach() for k, t in leaves.items()}
    E = torch.empty(0, device="cuda")
    cams = cams or [cam]
    H, W = cams[0].image_height, cams[0].image_width
    bg = torch.tensor([0.1, 0.4, 0.7], device="cuda")
    vm = torch.stack([c.viewmatrix for c in cams]).cuda()
    pm = torch.stack([c.projmatrix for c in cams]).cuda()
    cp = torch.stack([c.campos for c in cams]).cuda()
    table = [(c.tanfovx, c.tanfovy, c.cx, c.cy) for c in cams]
    cots = [cot] if V == 1 else cot
    stack = lambda j: torch.stack([c[j] for c in cots]).contiguous()
    ws = _lib.scratch(_lib.load().r3dg_raster_surface_grad_bytes(W, H, V), "cuda")
    if V == 1:
        c = cams[0]
        o = _C_raster.rasterize_gaussians(bg, d["means3D"], d["features"], E, d["opacities"], d["scales"], d["rotations"],
                                          1.0, E, vm[0], pm[0], c.tanfovx, c.tanfovy, c.cx, c.cy, H, W, d["shs"], 3,
                                          cp[0], False, True, False)
        cot, nbad = masked(cot, c, o[3], o[4])
        g = _C_raster.rasterize_gaussians_backward(bg, d["means3D"], d["features"], o[9], E, d["scales"],
                                                   d["rotations"], 1.0, E, vm[0], pm[0], c.tanfovx, c.tanfovy, *cot[:4],
                                                   d["shs"], 3, cp[0], o[10], o[0], o[11], o[12], True, False,
                                                   cam_grads=True, surface=(cot[4], cot[5], o[3], o[4], c.cx, c.cy),
                                                   surface_work=ws)
        opacity, depth = o[3][None], o[4][None]
    else:
        o = _C_raster.rasterize_views(bg[None].expand(V, 3).contiguous(), d["means3D"], d["features"], E, d["opacities"],
                                      d["scales"], d["rotations"], 1.0, E, vm, pm, table, H, W, d["shs"], 3, cp, False,
                                      True)
        cots = [masked(cots[v], cams[v], o[3][v], o[4][v])[0] for v in range(V)]
        g = _C_raster.rasterize_views_backward(bg[None].expand(V, 3).contiguous(), d["means3D"], d["features"], E,
                                               d["scales"], d["rotations"], 1.0, E, vm, pm, table, *(stack(j) for j in
                                                                                                     range(4)),
                                               d["shs"], 3, cp, o[10], o[11], o[12], True, cam_grads=True,
                                               surface=(stack(4), stack(5), o[3], o[4]), surface_work=ws)
        opacity, depth = o[3], o[4]
    torch.cuda.synchronize()
    HW = H * W
    f = ws.view(torch.float32)
    planes = f[:2 * V * HW].view(2, V, H, W)
    nblk = ((W + 31) // 32) * ((H + 7) // 8)
    off = (2 * V * HW * 4 + 255) // 256 * 64
    part = f[off:off + V * 9 * nblk].view(V, 9, nblk).double().sum(-1).view(V, 3, 3)
    if V == 1:
        print(f"[surface] {W}x{H}: normal cotangent zeroed on {nbad} ill-conditioned pixels of {HW}")
    return planes[0].clone(), planes[1].clone(), part, opacity, depth, g[9:], (cot if V == 1 else cots)


def truth(cam, cot, opacity, depth):
    """fp64 autograd of the restatement on the forward's fp32 images: (depth plane, opacity plane, dL/dV [3,3])."""
    H, W = cam.image_height, cam.image_width
    o64 = opacity.double().requires_grad_(True)
    d64 = depth.double().requires_grad_(True)
    V64 = cam.viewmatrix.cuda().double().requires_grad_(True)
    n, x = surface_normal(o64, d64, V64, W, H, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy)
    loss = (n * cot[4].double()).sum() + (x * cot[5].double()).sum()
    go, gd, gV = torch.autograd.grad(loss, [o64, d64, V64])
    return (cot[2].double() + gd).view(H, W), (cot[1].double() + go).view(H, W), gV[:3, :3]


def check_planes(tag, cam, cot, dplane, oplane, part, opacity, depth):
    want_d, want_o, want_V = truth(cam, cot, opacity, depth)
    assert torch.isfinite(dplane).all() and torch.isfinite(oplane).all(), tag
    ed = rel_l2(dplane.cpu().numpy(), want_d.cpu().numpy())
    eo = rel_l2(oplane.cpu().numpy(), want_o.cpu().numpy())
    ev = rel_l2(part.cpu().numpy(), want_V.cpu().numpy())
    print(f"[surface] {tag}: rel_l2 depth plane {ed:.2e}, opacity plane {eo:.2e}, dL/dV normal term {ev:.2e}")
    assert ed <= 1e-5 and eo <= 1e-5 and ev <= 1e-5, (tag, ed, eo, ev)


# ---- 1. off changes nothing ----------------------------------------------------------------------------------------
def test_off_and_untouched_change_nothing(det_mode):
    P, W, H, S = 100_000, 320, 240, 5
    leaves = make_leaves(P, S)
    cam = synth.make_camera(1, W, H, center_shift=True)
    cot = cotangents(H, W, S)
    today, n_today = one_view(leaves, cam, cot, False, touch=False)
    off, n_off = one_view(leaves, cam, cot, False, touch=True)          # the cotangents of normal / xyz are ignored
    on_untouched, n_on = one_view(leaves, cam, cot, True, touch=False)  # both cotangents None: no extra launch
    for got in (off, on_untouched):
        assert [k for k, t in today.items() if not bits_equal(got[k], t)] == []
    assert n_today == n_off == n_on
    on, n_surface = one_view(leaves, cam, cot, True, touch=True)
    assert n_surface == n_today + 2                                     # the surface pass and its camera sums
    assert not bits_equal(on["means3D"], today["means3D"])


# ---- 2. / 3. the adjoint is right, and the compositor consumes exactly its planes ----------------------------------
SCENES = {"shell-800": (300_000, 800, 800, 2, {}), "odd-333x250": (100_000, 333, 250, 5, dict(center_shift=True)),
          "strip-257x2": (50_000, 257, 2, 3, {}), "edge-background": (50_000, 320, 240, 6, dict(radius=9.0)),
          # narrow images: the column clamp with W = 2, and one-pixel-wide / -high images where one stencil vanishes
          # (n = 0: only surface_xyz has a gradient)
          "narrow-2x37": (20_000, 2, 37, 4, dict(center_shift=True)), "column-1x37": (20_000, 1, 37, 4, {}),
          "row-37x1": (20_000, 37, 1, 4, {})}


@pytest.mark.parametrize("name", list(SCENES))
def test_adjoint_planes_match_fp64_and_feed_the_compositor(name, det_mode):
    P, W, H, view, kw = SCENES[name]
    S = 5
    leaves = make_leaves(P, S)
    cam = synth.make_camera(view, W, H, **kw)
    cot = cotangents(H, W, S)
    dplane, oplane, part, opacity, depth, cam_c, cot = c_planes(leaves, cam, cot)
    if name == "edge-background":
        assert float((opacity == 0).float().mean()) > 0.05 and float((opacity > 0.5).float().mean()) > 0.01
    check_planes(name, cam, cot, dplane, oplane, part[0], opacity[0], depth[0])
    # the public API, surface gradients on, against surface gradients off fed with the planes read above
    on, _ = one_view(leaves, cam, cot, True)
    fed, _ = one_view(leaves, cam, cot, False, touch=False, plane_cot=(oplane[None], dplane[None]))
    assert [k for k, t in fed.items() if k != "viewmatrix" and not bits_equal(on[k], t)] == []
    assert bits_equal(on["viewmatrix"], cam_c[0])
    # dL/dviewmatrix: the projection's term (fed) plus the normal term, added once in fp32
    diff = on["viewmatrix"].double() - fed["viewmatrix"].double()
    ulp = 4 * torch.finfo(torch.float32).eps * torch.maximum(on["viewmatrix"].abs(), fed["viewmatrix"].abs()).double()
    tol = ulp[:3, :3] + 1e-5 * float(part[0].abs().max())
    assert bool(((diff[:3, :3] - part[0]).abs() <= tol).all())
    assert bool((diff[:, 3] == 0).all()) and bool((diff[3, :] == 0).all())


# ---- 4. several views ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("det", [True, False])
def test_views_planes_equal_one_view_calls(det):
    P, W, H, S, V = 100_000, 203, 150, 5, 3
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        leaves = make_leaves(P, S)
        cams = [synth.make_camera(k, W, H, center_shift=(k % 2 == 1)) for k in range(V)]
        cots = [cotangents(H, W, S, seed=40 + v) for v in range(V)]
        dp, op, part, opacity, depth, camg, cots = c_planes(leaves, None, cots, V=V, cams=cams)
        for v in range(V):
            d1, o1, p1, _, _, cam1, _ = c_planes(leaves, cams[v], cots[v])
            assert bits_equal(dp[v], d1[0]) and bits_equal(op[v], o1[0]), v
            assert torch.allclose(part[v], p1[0], rtol=1e-12, atol=0.0), v      # fp64 sums of the same partials
            if det:
                assert bits_equal(camg[0][v], cam1[0]), v
            if v == 0:
                check_planes("views", cams[v], cots[v], dp[v], op[v], part[v], opacity[v], depth[v])
        # the public API: per-view camera gradients, leaf gradients summed over the views
        vm = [c.viewmatrix.cuda().requires_grad_(True) for c in cams]
        settings = [settings_of(c, m, c.projmatrix.cuda(), c.campos.cuda()) for c, m in zip(cams, vm)]
        m2d = torch.zeros(V, P, 3, device="cuda", requires_grad=True)
        kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
        out = rasterize_views(leaves["means3D"], m2d, leaves["opacities"], settings=settings, surface_grads=True, **kw)
        loss = sum(sum((out[i][v] * c).sum() for i, c in zip(IMAGES + SURFACE, cots[v])) for v in range(V))
        gs = torch.autograd.grad(loss, [leaves["means3D"], leaves["opacities"]] + vm)
        ones = [one_view(leaves, cams[v], cots[v], True)[0] for v in range(V)]
        for k, name in enumerate(("means3D", "opacities")):
            want = sum(o[name] for o in ones)
            e = rel_l2(gs[k].cpu().numpy(), want.cpu().numpy())
            assert e <= (1e-6 if det else 1e-4), (name, e)
        for v in range(V):
            if det:
                assert bits_equal(gs[2 + v], ones[v]["viewmatrix"]), v
            else:
                assert rel_l2(gs[2 + v].cpu().numpy(), ones[v]["viewmatrix"].cpu().numpy()) <= 1e-4, v
    finally:
        torch.use_deterministic_algorithms(prev)


def test_one_view_rasterize_views_equals_gaussian_rasterizer(det_mode):
    """rasterize_views with a single setting runs the one-view library call: its surface adjoint must use that
    setting's principal point (here off-centre) and give GaussianRasterizer's gradients, bit for bit in the
    deterministic mode (both make the same library call)."""
    P, W, H, S = 100_000, 240, 180, 5
    leaves = make_leaves(P, S)
    cam = synth.make_camera(1, W, H, center_shift=True)
    cot = cotangents(H, W, S, seed=13)
    want, _ = one_view(leaves, cam, cot, True)
    vm = cam.viewmatrix.cuda().requires_grad_(True)
    m2d = torch.zeros(1, P, 3, device="cuda", requires_grad=True)
    kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
    out = rasterize_views(leaves["means3D"], m2d, leaves["opacities"],
                          settings=[settings_of(cam, vm, cam.projmatrix.cuda(), cam.campos.cuda())], surface_grads=True,
                          **kw)
    loss = sum((out[i][0] * c).sum() for i, c in zip(IMAGES + SURFACE, cot))
    names = list(leaves) + ["means2D", "viewmatrix"]
    gs = dict(zip(names, torch.autograd.grad(loss, list(leaves.values()) + [m2d, vm])))
    gs["means2D"] = gs["means2D"][0]
    for k in names:
        assert torch.isfinite(gs[k]).all(), k
        e = rel_l2(gs[k].cpu().numpy(), want[k].cpu().numpy())
        assert e <= 1e-6, (k, e)
    assert [k for k in names if not bits_equal(gs[k], want[k])] == []


# ---- 5. reproducibility and the deferred-count repair -------------------------------------------------------------
def test_reproducible_and_deferred_overflow_repair(det_mode):
    P, W, H, S = 50_000, 256, 192, 5
    leaves = make_leaves(P, S)
    cam = synth.make_camera(3, W, H)
    cot = cotangents(H, W, S)
    a, _ = one_view(leaves, cam, cot, True)
    b, _ = one_view(leaves, cam, cot, True)
    assert [k for k, t in a.items() if not bits_equal(b[k], t)] == []

    # deferred count: learn the instance counts on the same scene with small Gaussians, then boost the scales 20x so
    # that the speculative binning buffer (_HEADROOM = 1) overflows and the backward re-runs the forward
    P2, W2, H2 = 3000, 160, 120
    base = make_leaves(P2, S, seed=2)
    big = dict(base, scales=(base["scales"].detach() * 20.0).requires_grad_(True))
    cam2 = synth.make_camera(2, W2, H2)
    cot2 = cotangents(H2, W2, S, seed=9)
    _C_raster._state.clear()
    want, _ = one_view(big, cam2, cot2, True)                           # synchronous path: the truth
    _C_raster._state.clear()
    set_deferred_count(True)
    old = _C_raster._HEADROOM
    try:
        _C_raster._HEADROOM = 1.0
        for i in range(_C_raster._LEARN + 1):
            one_view(base, synth.make_camera(i % 8, W2, H2), cot2, True)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            got, _ = one_view(big, cam2, cot2, True)
        assert any("re-run" in str(x.message) for x in w), [str(x.message) for x in w]
        for k, t in want.items():
            e = rel_l2(got[k].cpu().numpy(), t.cpu().numpy())
            assert e <= 1e-6, (k, e)
    finally:
        _C_raster._HEADROOM = old
        set_deferred_count(False)
        _C_raster._state.clear()


# ---- 6. a two-way depth-normal consistency loss -------------------------------------------------------------------
def test_two_way_depth_normal_consistency():
    """neilf-shaped: S = 16 features whose channels 0:3 hold the rendered normal; the loss pulls the pseudo-normal and
    the normal feature towards each other.  Detaching the pseudo-normal (the reference's loss) must give a different
    means3D gradient; both are finite."""
    P, W, H, S = 200_000, 400, 300, 16
    sc = synth.make_scene(P, seed=4, S=S)
    feats = sc.features.clone()
    feats[:, 0:3] = sc.normals
    leaves = dict(means3D=sc.means3D, opacities=sc.opacities, shs=sc.shs, scales=sc.scales, rotations=sc.rotations,
                  features=feats)
    leaves = {k: v.cuda().contiguous().requires_grad_(True) for k, v in leaves.items()}
    cam = synth.make_camera(6, W, H)

    def grad(detach):
        vm, pm, cp = (t.cuda() for t in (cam.viewmatrix, cam.projmatrix, cam.campos))
        m2d = torch.zeros(P, 3, device="cuda", requires_grad=True)
        out = GaussianRasterizer(settings_of(cam, vm, pm, cp), surface_grads=True)(
            leaves["means3D"], m2d, leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"],
            rotations=leaves["rotations"], features=leaves["features"])
        opacity, normal_feat, pseudo = out[3], out[5][0:3], out[6]
        n = torch.nn.functional.normalize(normal_feat, dim=0)
        mask = (opacity > 0.5).float()
        p = pseudo.detach() if detach else pseudo
        loss = ((1.0 - (n * p).sum(0, keepdim=True)) * mask).mean()
        return torch.autograd.grad(loss, [leaves["means3D"], leaves["features"]])

    two_way, one_way = grad(False), grad(True)
    for g in two_way + one_way:
        assert torch.isfinite(g).all()
    assert float((two_way[0] - one_way[0]).abs().max()) > 0
    assert float(two_way[0].abs().max()) > 0
    e = rel_l2(two_way[1].cpu().numpy(), one_way[1].cpu().numpy())
    assert e < 1e-3                                                     # the feature's own term is unchanged
