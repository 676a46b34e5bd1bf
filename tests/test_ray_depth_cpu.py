"""The ray-depth rasterizer mode without a GPU: the fp64 closed form of the depth plane that the GPU tests use as their
truth (against a brute-force maximisation along the pixel's line, central differences and autograd, and its
perspective limit), the C layer's sizes and refusals with the mode on, and the host layer's plumbing of the flag."""
import ctypes
import inspect

import pytest
import torch

import aa_oracle
import proj64
import raydepth64
from helpers import fake_raster_library
from relightable3dgaussian_b200 import _C_raster, _lib, synth
from relightable3dgaussian_b200 import rasterizer as R

FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued


def _scene(P=16, seed=0):
    sc = synth.make_scene(P, "shell-v1", seed, 0)
    cam = synth.make_camera(1, 320, 240)
    c64 = proj64.Camera(cam.viewmatrix, cam.projmatrix, cam.campos, 320, 240, cam.tanfovx, cam.tanfovy)
    d = lambda t: t.double().clone()                                               # noqa: E731
    return d(sc.means3D), aa_oracle.cov3d_of(d(sc.scales) * 4.0, d(sc.rotations)), c64


def _inside(m, cam):
    """Rows whose projected centre is inside the frustum clamp (the plane is smooth there)."""
    t = m @ cam.V[:3, :3] + cam.V[3, :3]
    return bool((t[0] / t[2]).abs() < 1.2 * cam.tanfovx and (t[1] / t[2]).abs() < 1.2 * cam.tanfovy)


def test_closed_form_is_the_peak_along_the_pixel_line():
    """tz + p . offset is where the affine frame's filtered joint density peaks along the pixel's line."""
    m, sig, cam = _scene()
    n = 0
    for i in range(m.shape[0]):
        if not _inside(m[i], cam):
            continue
        p = raydepth64.plane(m[i], sig[i], cam, linearised=False)
        K, tz = raydepth64.joint(m[i], sig[i], cam)
        for off in ((0.0, 0.0), (3.0, -2.0), (-7.5, 4.25)):
            want = raydepth64.brute_peak(m[i], sig[i], cam, off)
            got = tz + p[0] * off[0] + p[1] * off[1]
            assert abs(float(got - want)) <= 1e-6 * float(torch.sqrt(K[2, 2])) + 1e-12, (i, off)
        n += 1
    assert n >= 8


def test_closed_form_matches_finite_differences_and_autograd():
    """d p / d (means3D, Sigma, viewmatrix) by autograd against central differences, and the plane depth zeroes the
    derivative of the joint log density in z (the conditional mean)."""
    m, sig, cam = _scene(P=6, seed=3)
    for i in range(m.shape[0]):
        if not _inside(m[i], cam):
            continue
        mi = m[i].clone().requires_grad_(True)
        si = sig[i].clone().requires_grad_(True)
        V = cam.V.clone().requires_grad_(True)

        def f(mm, ss, VV):
            c = proj64.Camera(VV, cam.P, cam.campos, cam.W, cam.H, cam.tanfovx, cam.tanfovy)
            return raydepth64.plane(mm, ss, c, linearised=False)
        for k in range(2):
            g = torch.autograd.grad(f(mi, si, V)[k], (mi, si, V))
            for x, gx in zip((mi, si, V), g):
                flat = x.detach().reshape(-1)
                for j in range(flat.numel()):
                    h = 1e-6 * max(1.0, abs(float(flat[j])))
                    xp, xm = flat.clone(), flat.clone()
                    xp[j] += h
                    xm[j] -= h
                    args = [mi.detach(), si.detach(), V.detach()]
                    idx = [t is x for t in (mi, si, V)].index(True)
                    args[idx] = xp.view(x.shape)
                    fp = f(*args)[k]
                    args[idx] = xm.view(x.shape)
                    fm = f(*args)[k]
                    fd = float((fp - fm) / (2 * h))
                    assert abs(fd - float(gx.reshape(-1)[j])) <= 1e-5 * (abs(fd) + 1e-3), (i, k, j)
        # the conditional mean: d/dz of the quadratic form vanishes at z = tz + p . off
        K, tz = raydepth64.joint(m[i], sig[i], cam)
        p = raydepth64.plane(m[i], sig[i], cam, linearised=False)
        off = torch.tensor([2.0, -1.5], dtype=torch.float64)
        z = (tz + p @ off).detach().requires_grad_(True)
        v = torch.cat([off, (z - tz)[None]])
        (q,) = torch.autograd.grad(v @ torch.linalg.inv(K) @ v, z)
        assert abs(float(q)) <= 1e-9 * float(1 / K[2, 2]), i


def test_plane_approaches_the_perspective_peak():
    """Without the screen filter, the affine plane's depth at one screen sigma from the centre approaches the exact
    peak of the 3D Gaussian along the perspective ray as the Gaussian shrinks relative to its depth: the error, in
    units of the Gaussian's depth extent, falls linearly with size / depth."""
    f = 300.0
    cam = proj64.Camera(torch.eye(4), torch.eye(4), torch.zeros(3), 2 * f, 2 * f, 1.0, 1.0)   # h = f, centre at 0
    q = torch.tensor([[0.9, 0.3, -0.2, 0.25]], dtype=torch.float64)
    mc = torch.tensor([0.4, -0.3, 5.0], dtype=torch.float64)
    errs = []
    for s in (0.2, 0.1, 0.05, 0.025):
        sig = aa_oracle.cov3d_of(torch.tensor([[s, 0.6 * s, 0.05 * s]], dtype=torch.float64), q)[0]   # a flat disc
        p = raydepth64.plane(mc, sig, cam, dilation=0.0, linearised=False)
        T, tz = raydepth64._T(mc, cam)
        C = T @ sig @ T.T
        off = torch.sqrt(C[0, 0]) * torch.tensor([1.0, 0.0], dtype=torch.float64)    # one screen sigma in x
        u = f * mc[:2] / mc[2] + off
        ray = torch.cat([u / f, torch.ones(1, dtype=torch.float64)])
        exact = raydepth64.perspective_peak(mc, sig, ray)
        affine = tz + p @ off
        errs.append(float((affine - exact).abs() / torch.sqrt(sig[2, 2])))
    for a, b in zip(errs, errs[1:]):
        assert b <= 0.6 * a, errs                  # halving the size at least nearly halves the relative error
    assert errs[-1] < 5e-3, errs


def test_sizes_grow_in_the_mode_only():
    lib = _lib.load()
    for P, S, V in ((1000, 5, 1), (1000, 16, 3), (0, 0, 1)):
        base = lib.r3dg_raster_views_geom_bytes(P, S, V)
        rd = lib.r3dg_raster_ray_depth_geom_bytes(P, S, V)
        # a record and a gradient row 16 B wider each (two regions, each rounded up to 256 B), and one 256-byte block
        assert abs(rd - base - 2 * 16 * max(P, 1) * V - 256) <= 2 * 256, (P, S, V)
    assert lib.r3dg_raster_ray_depth_geom_bytes(10, 5, 0) == lib.r3dg_raster_ray_depth_geom_bytes(10, 5, 1)
    # always larger than the default layout: a host tells a buffer's mode from its size
    for P in (0, 1, 2, 3, 7, 15, 16, 17, 63, 64, 65, 100, 1000, 4097):
        for S in (0, 1, 5, 16, 24, 33):
            for V in (1, 2, 3):
                assert lib.r3dg_raster_ray_depth_geom_bytes(P, S, V) > lib.r3dg_raster_views_geom_bytes(P, S, V)
    assert lib.r3dg_raster_views_geom_bytes(1000, 5, 1) == lib.r3dg_raster_geom_bytes(1000, 5)
    # gradient rows: 4 more accumulators per row, 24 B + 2 flag bits each (two regions rounded up to 256 B)
    assert lib.r3dg_raster_ray_depth_bwd_det_bytes(1000, 5) - lib.r3dg_raster_bwd_det_bytes(1000, 5) in range(96_000 + 1_000 - 512, 96_000 + 1_000 + 512)


def _fwd_args(lib, P=100, S=5, W=64, H=48):
    a = _lib.RasterFwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_ray_depth_geom_bytes(P, S, 1)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(W, H)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.means3D = a.opacities = a.shs = a.scales = a.rotations = FAKE
    a.ray_depth = 1
    return a


def _bwd_args(lib, P=100, S=5, W=64, H=48):
    a = _lib.RasterBwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_ray_depth_geom_bytes(P, S, 1)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(W, H)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.dL_dmeans2D = a.dL_dopacity = a.dL_dmeans3D = a.dL_dcov3D = a.dL_dscales = a.dL_drotations = FAKE
    a.ray_depth = 1
    return a


@pytest.mark.parametrize("flaw", ["geom-of-the-default-mode", "geom-one-byte-short", "det-no-work"])
def test_forward_refusals_with_the_mode_on(flaw):
    lib = _lib.load()
    a = _fwd_args(lib)
    if flaw == "geom-of-the-default-mode":
        a.geom_bytes = lib.r3dg_raster_geom_bytes(100, 5)
    elif flaw == "geom-one-byte-short":
        a.geom_bytes -= 1
    elif flaw == "det-no-work":
        a.deterministic = 1
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001, flaw


@pytest.mark.parametrize("flaw", ["geom-of-the-default-mode", "det-work-of-the-default-mode",
                                  "det-work-without-absgrad-part"])
def test_backward_refusals_with_the_mode_on(flaw):
    lib = _lib.load()
    a = _bwd_args(lib)
    if flaw == "geom-of-the-default-mode":
        a.geom_bytes = lib.r3dg_raster_geom_bytes(100, 5)
    elif flaw == "det-work-of-the-default-mode":
        a.deterministic = 1
        a.det_work, a.det_work_bytes = FAKE, lib.r3dg_raster_bwd_det_bytes(100, 5)
    elif flaw == "det-work-without-absgrad-part":
        a.deterministic = 1
        a.dL_dmeans2D_abs = FAKE
        a.det_work, a.det_work_bytes = FAKE, lib.r3dg_raster_ray_depth_bwd_det_bytes(100, 5)
    assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001, flaw


def test_field_sits_with_the_other_mode_flags():
    tail = ["antialiasing", "deterministic", "det_work", "det_work_bytes"]
    assert [f[0] for f in _lib.RasterFwdArgs._fields_[-5:]] == ["ray_depth"] + tail
    assert [f[0] for f in _lib.RasterBwdArgs._fields_[-6:]] == ["ray_depth", "dL_dmeans2D_abs"] + tail


def test_keyword_defaults_are_off():
    for fn in (R.rasterize_gaussians, R.rasterize_views):
        assert inspect.signature(fn).parameters["ray_depth"].default is False, fn.__name__
    assert inspect.signature(R.GaussianRasterizer.__init__).parameters["ray_depth"].default is False
    # the library entry points: None = the process default (forward) or the forward's mode (backward)
    for fn in (_C_raster.rasterize_gaussians, _C_raster.rasterize_gaussians_backward, _C_raster.rasterize_views,
               _C_raster.rasterize_views_backward):
        assert inspect.signature(fn).parameters["ray_depth"].default is None, fn.__name__
    assert _C_raster._fwd_ray_depth(None) is False
    R.set_ray_depth(True)
    try:
        assert _C_raster._fwd_ray_depth(None) is True and _C_raster._fwd_ray_depth(False) is False
    finally:
        R.set_ray_depth(False)


def test_set_ray_depth_round_trips_through_the_forward(monkeypatch):
    calls = fake_raster_library(monkeypatch)
    rs, lv = _settings()
    P = lv["means3D"].shape[0]

    def render(**kw):
        R.GaussianRasterizer(rs, **kw)(means3D=lv["means3D"], means2D=torch.zeros(P, 3), opacities=lv["opacities"],
                                       shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"])
    render()
    R.set_ray_depth(True)
    try:
        render()
    finally:
        R.set_ray_depth(False)
    render()
    render(ray_depth=True)
    assert [kw.get("ray_depth") for _, kw in calls] == [None, True, None, True]


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


@pytest.mark.parametrize("how", ["off", "keyword", "process-default"])
def test_host_layer_passes_the_flag(monkeypatch, how):
    """GaussianRasterizer and rasterize_views hand `ray_depth=True` to the library call when the mode is on (by keyword
    or set_ray_depth), and call it exactly as before (no such keyword) when it is off."""
    seen = []

    def fake(*args, **kw):
        seen.append(kw)
        raise _Stop()
    monkeypatch.setattr(R._C, "rasterize_gaussians", fake)
    monkeypatch.setattr(R._C, "rasterize_views", fake)
    rs, lv = _settings()
    P = lv["means3D"].shape[0]
    kw = {"ray_depth": True} if how == "keyword" else {}
    R.set_ray_depth(how == "process-default")
    try:
        with pytest.raises(_Stop):
            R.GaussianRasterizer(rs, **kw)(means3D=lv["means3D"], means2D=torch.zeros(P, 3),
                                           opacities=lv["opacities"], shs=lv["shs"], scales=lv["scales"],
                                           rotations=lv["rotations"])
        with pytest.raises(_Stop):
            R.rasterize_views(lv["means3D"], torch.zeros(2, P, 3), lv["opacities"], settings=[rs, rs], shs=lv["shs"],
                              scales=lv["scales"], rotations=lv["rotations"], **kw)
    finally:
        R.set_ray_depth(False)
    assert [k.get("ray_depth") for k in seen] == ([None, None] if how == "off" else [True, True])


def test_library_backward_gets_the_flag(monkeypatch):
    """The autograd node hands the forward's flag to the library backward, also for the appearance-only backward (its
    work buffers have the mode's layout)."""
    calls = fake_raster_library(monkeypatch)
    rs, lv = _settings()
    P = lv["means3D"].shape[0]
    out = R.GaussianRasterizer(rs, ray_depth=True)(means3D=lv["means3D"], means2D=torch.zeros(P, 3),
                                                   opacities=lv["opacities"], shs=lv["shs"].requires_grad_(True),
                                                   scales=lv["scales"], rotations=lv["rotations"])
    out[2].sum().backward()
    name, kw = calls[-1]
    assert name == "rasterize_gaussians_backward"
    assert kw.get("ray_depth") is True and kw.get("geometry") is False


def test_debug_snapshot_records_the_flag(monkeypatch, tmp_path):
    def fake(*args, **kw):
        raise _Stop()
    monkeypatch.setattr(R._C, "rasterize_gaussians", fake)
    monkeypatch.chdir(tmp_path)
    rs, lv = _settings(debug=True)
    P = lv["means3D"].shape[0]
    with pytest.raises(_Stop):
        R.rasterize_gaussians(lv["means3D"], torch.zeros(P, 3), torch.zeros(P, 0), lv["shs"], torch.Tensor([]),
                              lv["opacities"], lv["scales"], lv["rotations"], torch.Tensor([]), rs, ray_depth=True)
    saved = torch.load(tmp_path / "snapshot_fw.dump", weights_only=False)
    assert saved[-1]["ray_depth"] is True
