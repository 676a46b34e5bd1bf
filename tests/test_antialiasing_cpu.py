"""The antialiased rasterizer mode without a GPU: the fp64 closed form of the opacity factor rho that the GPU tests use
as their truth (against central finite differences, and its limits), the cancellation-free derivative forms of the
projection backward, the C layer's refusals with the mode on, and the host layer's plumbing of the flag."""
import ctypes

import pytest
import torch

import aa_oracle
from relightable3dgaussian_b200 import _lib, synth
from relightable3dgaussian_b200 import rasterizer as R

FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued


def _scene(P=24, seed=0, boost=1.0):
    sc = synth.make_scene(P, "shell-v1", seed, 0)
    cam = synth.make_camera(1, 320, 240)
    d = lambda t: t.double().clone()
    return d(sc.means3D), d(sc.scales) * boost, d(sc.rotations), cam


def _rho(cam, **kw):
    return aa_oracle.rho(viewmatrix=kw.pop("viewmatrix", cam.viewmatrix.double()), W=cam.image_width,
                         H=cam.image_height, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, **kw)


def test_closed_form_matches_finite_differences():
    """d rho / d (means3D, scales, rotations | cov3D, viewmatrix) of the closed form against central differences, on
    Gaussians away from the floor and the frustum clamp (where rho is not differentiable)."""
    means3D, scales, rotations, cam = _scene()
    vm = cam.viewmatrix.double()
    r = _rho(cam, means3D=means3D, scales=scales, rotations=rotations)
    keep = (r > 0.02) & (r < 0.999)
    assert int(keep.sum()) >= 8
    m, s, q = means3D[keep], scales[keep], rotations[keep]
    f = lambda m, s, q, v: _rho(cam, means3D=m, scales=s, rotations=q, viewmatrix=v)
    assert torch.autograd.gradcheck(f, tuple(t.clone().requires_grad_(True) for t in (m, s, q, vm)), eps=1e-7,
                                    atol=1e-6, rtol=1e-5)
    c6 = aa_oracle.cov3d_of(s, q)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].contiguous()
    g = lambda m, c, v: _rho(cam, means3D=m, cov3D=c, viewmatrix=v)
    assert torch.autograd.gradcheck(g, tuple(t.clone().requires_grad_(True) for t in (m, c6, vm)), eps=1e-9,
                                    atol=1e-6, rtol=1e-5)
    # the same rho from the covariance given either way
    assert torch.allclose(g(m, c6, vm), f(m, s, q, vm), rtol=1e-12, atol=0)


def test_cancellation_free_derivatives():
    """The projection backward's dr/da = 0.3 (c0 c1 + b^2) / det1^2, dr/dc = 0.3 (a0 a1 + b^2) / det1^2 and
    dr/db = -2 b (0.3 (a0 + c0) + 0.09) / det1^2 are the derivatives of r = det0 / det1."""
    g = torch.Generator().manual_seed(3)
    L = torch.randn(200, 2, 2, generator=g, dtype=torch.float64) * torch.logspace(-3, 2, 200, dtype=torch.float64)[:, None, None]
    C = L @ L.transpose(1, 2)
    a0, b, c0 = (C[:, 0, 0].clone().requires_grad_(True), C[:, 0, 1].clone().requires_grad_(True),
                 C[:, 1, 1].clone().requires_grad_(True))
    r = aa_oracle.ratio(a0, b, c0)
    assert bool((r > 0).all())
    want = torch.autograd.grad(r.sum(), (a0, b, c0))
    got = aa_oracle.ratio_grad(a0.detach(), b.detach(), c0.detach())
    for w, x in zip(want, got):
        torch.testing.assert_close(x, w, rtol=1e-10, atol=1e-300)


def test_limits():
    """rho -> 1 for Gaussians much larger than a pixel, ~ sqrt(det0) / 0.3 for tiny ones, and the floor 0.005 with no
    gradient where det0 <= 0."""
    means3D, scales, rotations, cam = _scene(boost=1e3)
    big = _rho(cam, means3D=means3D, scales=scales, rotations=rotations)
    assert bool((big > 0.999).all()), big.min()
    tiny_s = scales * 1e-4
    tiny = _rho(cam, means3D=means3D, scales=tiny_s, rotations=rotations)
    a0, b, c0 = aa_oracle.cov2d(means3D, aa_oracle.cov3d_of(tiny_s, rotations), cam.viewmatrix.double(),
                                cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy)
    approx = (a0 * c0 - b * b).clamp_min(0).sqrt() / 0.3
    above = (approx > 0.006) & (a0 + c0 < 0.01)     # both variances well below the 0.3 px^2 dilation
    assert bool(above.any())
    torch.testing.assert_close(tiny[above], approx[above], rtol=0.02, atol=0)
    # det0 <= 0: a rank-1 (needle) covariance, a zero one and an indefinite one
    c6 = torch.tensor([[1.0, 0.0, 0.0, 0.0, 0.0, 0.0], [0.0] * 6, [1.0, 0.0, 0.0, -1.0, 0.0, 0.5]],
                      dtype=torch.float64, requires_grad=True)
    m = torch.tensor([[0.0, 0.0, 4.0]] * 3, dtype=torch.float64, requires_grad=True)
    vm = torch.eye(4, dtype=torch.float64, requires_grad=True)
    floor = aa_oracle.rho(m, vm, 320, 240, 0.5, 0.4, cov3D=c6)
    assert floor.tolist() == [0.005] * 3
    for gr in torch.autograd.grad(floor.sum(), (m, c6, vm)):
        assert bool((gr == 0).all())


def _fwd_args(lib, P=100, S=5, W=64, H=48):
    a = _lib.RasterFwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(W, H)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.means3D = a.opacities = a.shs = a.scales = a.rotations = FAKE
    a.antialiasing = 1
    return a


def _bwd_args(lib, P=100, S=5, W=64, H=48):
    a = _lib.RasterBwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(W, H)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.antialiasing = 1
    return a


def test_field_sits_before_the_deterministic_fields():
    for cls in (_lib.RasterFwdArgs, _lib.RasterBwdArgs):
        assert [f[0] for f in cls._fields_[-4:]] == ["antialiasing", "deterministic", "det_work", "det_work_bytes"]


@pytest.mark.parametrize("flaw", ["no-colour", "both-colours", "no-covariance", "det-no-work", "bad-size", "bad-views"])
def test_forward_refusals_with_the_mode_on(flaw):
    lib = _lib.load()
    a = _fwd_args(lib)
    if flaw == "no-colour":
        a.shs = None
    elif flaw == "both-colours":
        a.colors_precomp = FAKE
    elif flaw == "no-covariance":
        a.scales = None
    elif flaw == "det-no-work":
        a.deterministic = 1
    elif flaw == "bad-size":
        a.W = 0
    elif flaw == "bad-views":
        a.V = 3                       # no camera table
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001, flaw


@pytest.mark.parametrize("flaw", ["partial-geometry", "partial-camera", "small-camera-work", "det-no-work",
                                  "surface-no-images"])
def test_backward_refusals_with_the_mode_on(flaw):
    lib = _lib.load()
    a = _bwd_args(lib)
    a.dL_dmeans2D = a.dL_dopacity = a.dL_dmeans3D = a.dL_dcov3D = a.dL_dscales = a.dL_drotations = FAKE
    if flaw == "partial-geometry":
        a.dL_dcov3D = None
    elif flaw == "partial-camera":
        a.dL_dviewmatrix = FAKE
    elif flaw == "small-camera-work":
        a.dL_dviewmatrix = a.dL_dprojmatrix = a.dL_dcampos = FAKE
        a.cam_work, a.cam_work_bytes = FAKE, lib.r3dg_raster_cam_grad_bytes(100, 1) - 1
    elif flaw == "det-no-work":
        a.deterministic = 1
    elif flaw == "surface-no-images":
        a.dL_dout_normal = FAKE
    assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001, flaw


class _Stop(Exception):
    pass


def _settings(debug=False, P=7, H=4, W=5):
    rs = R.GaussianRasterizationSettings(H, W, 1.0, 1.0, 2.5, 2.0, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3,
                                         torch.zeros(3), False, True, True, debug)
    g = torch.Generator().manual_seed(0)
    leaves = dict(means3D=torch.randn(P, 3, generator=g), opacities=torch.rand(P, 1, generator=g),
                  shs=torch.randn(P, 16, 3, generator=g), scales=torch.rand(P, 3, generator=g),
                  rotations=torch.randn(P, 4, generator=g))
    return rs, leaves


@pytest.mark.parametrize("on", [False, True])
def test_host_layer_passes_the_flag(monkeypatch, on):
    """GaussianRasterizer and rasterize_views hand `antialiasing=True` to the library call when the mode is on, and
    call it exactly as before (no such keyword) when it is off."""
    seen = []

    def fake(*args, **kw):
        seen.append(kw)
        raise _Stop()
    monkeypatch.setattr(R._C, "rasterize_gaussians", fake)
    monkeypatch.setattr(R._C, "rasterize_views", fake)
    rs, lv = _settings()
    P = lv["means3D"].shape[0]
    with pytest.raises(_Stop):
        R.GaussianRasterizer(rs, antialiasing=on)(means3D=lv["means3D"], means2D=torch.zeros(P, 3),
                                                  opacities=lv["opacities"], shs=lv["shs"], scales=lv["scales"],
                                                  rotations=lv["rotations"])
    with pytest.raises(_Stop):
        R.rasterize_views(lv["means3D"], torch.zeros(2, P, 3), lv["opacities"], settings=[rs, rs], shs=lv["shs"],
                          scales=lv["scales"], rotations=lv["rotations"], antialiasing=on)
    assert [k.get("antialiasing") for k in seen] == ([True, True] if on else [None, None])


def test_debug_snapshot_records_the_flag(monkeypatch, tmp_path):
    def fake(*args, **kw):
        raise _Stop()
    monkeypatch.setattr(R._C, "rasterize_gaussians", fake)
    monkeypatch.chdir(tmp_path)
    rs, lv = _settings(debug=True)
    P = lv["means3D"].shape[0]
    with pytest.raises(_Stop):
        R.rasterize_gaussians(lv["means3D"], torch.zeros(P, 3), torch.zeros(P, 0), lv["shs"], torch.Tensor([]),
                              lv["opacities"], lv["scales"], lv["rotations"], torch.Tensor([]), rs, antialiasing=True)
    saved = torch.load(tmp_path / "snapshot_fw.dump", weights_only=False)
    assert saved[-1]["antialiasing"] is True
