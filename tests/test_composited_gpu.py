"""Rows no pixel composited: the forward marks the composited rows (debug id `composited`), and the backward neither
zeroes nor reads any other row.  Their gradients are exactly +0 in every output, in the default and the deterministic
mode, with and without camera gradients, for one view and for several views that occlude different Gaussians; a
Gaussian hidden behind an opaque wall gets +0 and the same Gaussian in front of it matches the CPU oracle."""
import contextlib

import numpy as np
import pytest
import torch

from helpers import case_inputs, npy, oracle_kwargs, rel_l2
from relightable3dgaussian_b200 import synth
from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_views)
import test_raster_gpu as tr

pytestmark = pytest.mark.gpu
LEAVES = ("means3D", "opacities", "scales", "rotations", "shs", "features")


@contextlib.contextmanager
def deterministic(on):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev)


@pytest.fixture(scope="module")
def C():
    from relightable3dgaussian_b200 import _C_raster
    assert torch.cuda.is_available()
    return _C_raster


def settings_of(cam, deg, cam_grads, bg):
    vm, pm, cp = (t.cuda().contiguous().requires_grad_(cam_grads) for t in (cam.viewmatrix, cam.projmatrix, cam.campos))
    return GaussianRasterizationSettings(cam.image_height, cam.image_width, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                         bg.cuda(), 1.0, vm, pm, deg, cp, False, True, True, False)


def leaves_of(sc, deg):
    d = dict(means3D=sc.means3D, opacities=sc.opacities, scales=sc.scales, rotations=sc.rotations,
             shs=sc.shs[:, : (deg + 1) ** 2].contiguous(), features=sc.features)
    return {k: v.cuda().contiguous().requires_grad_(True) for k, v in d.items() if v is not None and v.numel()}


def render_and_grads(settings, leaves, seed=3, retain=False):
    """Forward of one view (settings) or several (a list) with a random linear loss; returns (out weights [V, P],
    {name: gradient}, the loss and its inputs for a second backward).  Gradients: the leaves, means2D and, when the
    settings' cameras require grad, the camera matrices."""
    many = isinstance(settings, list)
    P = leaves["means3D"].shape[0]
    m2d = torch.zeros((len(settings), P, 3) if many else (P, 3), device="cuda", requires_grad=True)
    kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
    if many:
        out = rasterize_views(leaves["means3D"], m2d, leaves["opacities"], settings=settings, **kw)
    else:
        out = GaussianRasterizer(settings)(leaves["means3D"], m2d, leaves["opacities"], **kw)
    g = torch.Generator(device="cuda").manual_seed(seed)
    loss = sum((o * torch.randn(o.shape, device="cuda", generator=g)).sum() for o in out[2:6])
    names, inputs = list(leaves) + ["means2D"], list(leaves.values()) + [m2d]
    for v, s in enumerate(settings if many else [settings]):
        if s.viewmatrix.requires_grad:
            names += [f"viewmatrix{v}", f"projmatrix{v}", f"campos{v}"]
            inputs += [s.viewmatrix, s.projmatrix, s.campos]
    gs = torch.autograd.grad(loss, inputs, retain_graph=retain, allow_unused=True)
    weights = out[8].detach().reshape(len(settings) if many else 1, P)
    return weights, dict(zip(names, gs)), (loss, inputs)


def assert_plus_zero(name, t):
    assert t.numel() == 0 or (not t.any() and not torch.signbit(t).any()), name


def check_rows(weights, grads):
    """Rows composited in no view: every leaf gradient +0; means2D per view: +0 where the view did not composite."""
    live_any = (weights > 0).any(0)
    assert live_any.any() and not live_any.all()
    for n, t in grads.items():
        if n.rstrip("0123456789") in ("viewmatrix", "projmatrix", "campos"):
            assert torch.isfinite(t).all() and t.abs().sum() > 0, n
        elif n == "means2D":
            t = t.reshape(weights.shape[0], -1, 3)
            for v in range(weights.shape[0]):
                assert_plus_zero(f"means2D view {v}", t[v][weights[v] == 0])
                assert t[v][weights[v] > 0].abs().sum() > 0
        else:
            assert_plus_zero(n, t[~live_any])
            assert t[live_any].abs().sum() > 0, n


@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_flag_equals_positive_weight(C, det):
    sc, cam = case_inputs(300_000, 800, 800, 5, view=2)
    kw = oracle_kwargs(sc, cam, torch.tensor([0.0, 0.5, 1.0]))
    kw.update(shs=npy(sc.shs), scales=npy(sc.scales), rotations=npy(sc.rotations), features=npy(sc.features))
    with deterministic(det):
        o = tr.run_ours(C, **kw)
    flag = o["mid"]("composited").bool()
    w = o["weights"].reshape(-1)
    assert torch.equal(flag, w > 0)
    assert (o["radii"] > 0).sum() > flag.sum() > 0          # visible rows that no pixel composited exist


@pytest.mark.parametrize("cam_grads", [False, True], ids=["nocam", "cam"])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_rows_not_composited_get_plus_zero_one_view(det, cam_grads):
    sc, cam = case_inputs(300_000, 800, 800, 5, view=2)
    with deterministic(det):
        weights, grads, _ = render_and_grads(settings_of(cam, 3, cam_grads, torch.tensor([0.0, 0.5, 1.0])),
                                             leaves_of(sc, 3))
    check_rows(weights, grads)


@pytest.mark.parametrize("cam_grads", [False, True], ids=["nocam", "cam"])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_rows_not_composited_get_plus_zero_three_views(det, cam_grads):
    """Three cameras around the shell: each view composites a different front, so a row can be live in one view and
    not in the next (later views must leave the earlier views' sums as they are)."""
    sc = synth.make_scene(300_000, "shell-v1", 0, 5)
    cams = [synth.make_camera(k, 800, 800, center_shift=(k % 2 == 1)) for k in (0, 3, 5)]
    settings = [settings_of(c, 3, cam_grads, torch.tensor([0.1 * k, 0.5, 1.0])) for k, c in enumerate(cams)]
    with deterministic(det):
        weights, grads, _ = render_and_grads(settings, leaves_of(sc, 3))
    live = weights > 0
    assert (live.any(0) & ~live.all(0)).any()              # rows live in some views only
    check_rows(weights, grads)


def test_two_backwards_of_one_forward_bitwise_equal():
    """retain_graph: the composited rows are zeroed by every backward, so the second one does not accumulate."""
    sc, cam = case_inputs(300_000, 800, 800, 5, view=2)
    with deterministic(True):
        _, g1, (loss, inputs) = render_and_grads(settings_of(cam, 3, True, torch.tensor([0.0, 0.5, 1.0])),
                                                 leaves_of(sc, 3), retain=True)
        g2 = torch.autograd.grad(loss, inputs, allow_unused=True)
    for (n, a), b in zip(g1.items(), g2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), n


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_sh_degrees(deg):
    """Row widths of 12, 48 (bulk copies) and 3, 27 floats (transposed slab) with partly live CTAs."""
    sc, cam = case_inputs(100_000, 400, 400, 0, view=1)
    for det in (False, True):
        with deterministic(det):
            weights, grads, _ = render_and_grads(settings_of(cam, deg, False, torch.tensor([0.2, 0.2, 0.2])),
                                                 leaves_of(sc, deg))
        check_rows(weights, grads)
        assert grads["shs"].shape[1] == (deg + 1) ** 2


def _wall_scene(front):
    """Two layers of opaque Gaussians at depths 4.0 / 4.1 filling the view's centre, and one Gaussian G (the last row)
    on the axis at depth 3 (front) or 6 (behind the wall)."""
    cam = synth.make_axis_camera(128, 96)
    xs = torch.linspace(-0.8, 0.8, 33)
    gy, gx = torch.meshgrid(xs * 0.75, xs, indexing="ij")
    layer = torch.stack([gx.reshape(-1), gy.reshape(-1)], 1)
    n = layer.shape[0]
    means = torch.cat([torch.cat([layer, torch.full((n, 1), z)], 1) for z in (4.0, 4.1)] +
                      [torch.tensor([[0.03, -0.02, 3.0 if front else 6.0]])])
    P = means.shape[0]
    g = torch.Generator().manual_seed(7)
    scales = torch.full((P, 3), 0.06)
    scales[-1] = torch.tensor([0.05, 0.03, 0.04])
    rot = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=1)
    opac = torch.full((P, 1), 0.99)
    opac[-1] = 0.8
    shs = 0.5 * torch.randn(P, 16, 3, generator=g)
    feats = torch.rand(P, 5, generator=g)
    return cam, dict(means3D=means, opacities=opac, scales=scales, rotations=rot, shs=shs, features=feats)


@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_gaussian_behind_a_wall_and_in_front_of_it(C, det):
    from oracle import oracle
    for front in (False, True):
        cam, d = _wall_scene(front)
        bg = torch.tensor([0.3, 0.1, 0.6])
        kw = dict(means3D=npy(d["means3D"]), opacities=npy(d["opacities"]), viewmatrix=npy(cam.viewmatrix),
                  projmatrix=npy(cam.projmatrix), campos=npy(cam.campos), bg=npy(bg), W=cam.image_width,
                  H=cam.image_height, tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy)
        extra = dict(shs=npy(d["shs"]), scales=npy(d["scales"]), rotations=npy(d["rotations"]),
                     features=npy(d["features"]))
        rng = np.random.default_rng(11)
        cots = [rng.standard_normal((c, cam.image_height, cam.image_width)).astype(np.float32) for c in (3, 1, 1, 5)]
        with deterministic(det):
            o = tr.run_ours(C, cots=cots, **kw, **extra)
        flag = o["mid"]("composited").bool()
        assert o["radii"][-1] > 0 and bool(flag[-1]) == front
        assert torch.equal(flag, o["weights"].reshape(-1) > 0)
        if not front:
            for n, t in o["grads"].items():
                assert_plus_zero(n, t[-1])
            continue
        f = oracle.rasterize_forward(**kw, **extra)
        bk = {k: v for k, v in {**kw, **extra}.items() if k not in ("opacities", "cx", "cy")}
        gr = oracle.rasterize_backward(f, dL_dcolor=cots[0], dL_dopacity=cots[1], dL_ddepth=cots[2],
                                       dL_dfeature=cots[3], **bk)
        for n in tr.GRADS:
            ours, ref = npy(o["grads"][n])[-1], gr[n][-1]
            assert np.abs(ref).max() > 0, n
            assert rel_l2(ours, ref) < 1e-3, (n, rel_l2(ours, ref))
