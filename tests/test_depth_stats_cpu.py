"""The rasterizer's depth statistics without a GPU: the fp64 oracle's identities (depth2 against the pairwise
distortion, the median rule on hand-built lists, central differences), the C layer's sizes and refusals, and the host
layer's plumbing of the flag."""
import ctypes
import inspect

import pytest
import torch

import depthstats64 as ds64
from helpers import fake_raster_library
from relightable3dgaussian_b200 import _C_raster, _lib
from relightable3dgaussian_b200 import rasterizer as R

FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued


def test_distortion_is_opacity_times_depth2_minus_depth_squared():
    g = torch.Generator().manual_seed(0)
    alphas = torch.rand(64, 12, generator=g, dtype=torch.float64) * 0.9
    alphas[alphas < 0.05] = 0.0                                    # skipped entries
    w, T, valid = ds64.lists(alphas)
    d = 1.0 + 4.0 * torch.rand(64, 12, generator=g, dtype=torch.float64)
    d2, _, _ = ds64.stats(w, d, T, valid)
    A = torch.where(valid, w, torch.zeros_like(w)).sum(1)
    D = torch.where(valid, w * d, torch.zeros_like(w)).sum(1)
    torch.testing.assert_close(A * d2 - D * D, ds64.distortion(w, d, valid), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("case,alphas,want_pos", [
    ("crosses", [0.2, 0.3, 0.4, 0.5], 3),            # T before: 1, 0.8, 0.56, 0.336 -> the third takes T through 0.5
    ("never-crosses", [0.1, 0.1, 0.1], 3),          # T stays above 0.5: the last composited entry
    ("skips", [0.3, 0.0, 0.5, 0.2], 3),             # the skipped second entry is not a candidate
    ("first-entry", [0.6, 0.5, 0.5], 1),            # T before the second is 0.4: only the first had T > 0.5
    ("early-stop", [0.3, 0.99, 0.99, 0.99], 2),     # the third entry stops the pixel (T 0.007 -> 7e-5) and is not composited
    ("empty", [0.0, 0.0], 0),
])
def test_median_rule_on_hand_built_lists(case, alphas, want_pos):
    a = torch.tensor([alphas], dtype=torch.float64)
    w, T, valid = ds64.lists(a)
    d = torch.arange(1, a.shape[1] + 1, dtype=torch.float64)[None] * 10.0
    _, med, pos = ds64.stats(w, d, T, valid)
    assert int(pos[0]) == want_pos, (case, T, valid)
    assert float(med[0]) == (10.0 * want_pos if want_pos else 0.0)
    if case == "early-stop":
        assert bool(valid[0, 1]) and not bool(valid[0, 2:].any())


def test_oracle_gradients_match_central_differences():
    g = torch.Generator().manual_seed(3)
    alphas = 0.05 + 0.6 * torch.rand(8, 6, generator=g, dtype=torch.float64)
    d0 = 1.0 + 3.0 * torch.rand(8, 6, generator=g, dtype=torch.float64)
    g2, gm = torch.randn(8, generator=g, dtype=torch.float64), torch.randn(8, generator=g, dtype=torch.float64)

    def loss(a, d):
        w, T, valid = ds64.lists(a.detach())       # the lists' discrete decisions at the base point
        one = torch.where(valid, 1.0 - a, torch.ones_like(a))
        Tb = torch.cumprod(torch.cat([torch.ones_like(a[:, :1]), one[:, :-1]], 1), 1)
        d2, med, _ = ds64.stats(a * Tb, d, T, valid)
        return (d2 * g2).sum() + (med * gm).sum()
    a = alphas.clone().requires_grad_(True)
    d = d0.clone().requires_grad_(True)
    ga, gd = torch.autograd.grad(loss(a, d), (a, d))
    h = 1e-6
    for x, gx, which in ((alphas, ga, 0), (d0, gd, 1)):
        for idx in [(0, 0), (3, 2), (7, 5), (5, 1)]:
            xp, xm = x.clone(), x.clone()
            xp[idx] += h
            xm[idx] -= h
            args_p = (xp, d0) if which == 0 else (alphas, xp)
            args_m = (xm, d0) if which == 0 else (alphas, xm)
            fd = float((loss(*args_p) - loss(*args_m)) / (2 * h))
            assert abs(fd - float(gx[idx])) <= 1e-6 * (abs(fd) + 1.0), (which, idx, fd, float(gx[idx]))


def test_sizes_grow_with_the_flag_only():
    lib = _lib.load()
    for W, H in ((1, 1), (64, 48), (800, 800), (1920, 1080), (4100, 16)):
        for V in (1, 2, 5):
            base = lib.r3dg_raster_views_img_bytes(W, H, V)
            ds = lib.r3dg_raster_depth_stats_img_bytes(W, H, V)
            assert ds > base and ds % 256 == 0, (W, H, V)
            # the median positions (4 B per pixel) and one word per view, each region rounded up to 256 B
            assert ds - base <= 4 * W * H * V + 2 * 256 + 4 * V, (W, H, V)
            assert ds - base >= 4 * W * H * V
    assert lib.r3dg_raster_depth_stats_img_bytes(64, 48, 0) == lib.r3dg_raster_depth_stats_img_bytes(64, 48, 1)
    # the default layouts are those of the parent
    assert lib.r3dg_raster_views_img_bytes(800, 800, 1) == lib.r3dg_raster_img_bytes(800, 800) == 15461376


def _fwd_args(lib, P=100, S=5, W=64, H=48):
    a = _lib.RasterFwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_depth_stats_img_bytes(W, H, 1)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.means3D = a.opacities = a.shs = a.scales = a.rotations = FAKE
    a.depth_stats, a.out_depth2, a.out_median_depth = 1, FAKE, FAKE
    return a


def _bwd_args(lib, P=100, S=5, W=64, H=48):
    a = _lib.RasterBwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_depth_stats_img_bytes(W, H, 1)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.dL_dmeans2D = a.dL_dopacity = a.dL_dmeans3D = a.dL_dcov3D = a.dL_dscales = a.dL_drotations = FAKE
    a.depth_stats, a.dL_dout_depth2, a.dL_dout_median_depth = 1, FAKE, FAKE
    return a


@pytest.mark.parametrize("flaw", ["img-of-the-default-layout", "img-one-byte-short", "no-depth2", "no-median"])
def test_forward_refusals(flaw):
    lib = _lib.load()
    a = _fwd_args(lib)
    if flaw == "img-of-the-default-layout":
        a.img_bytes = lib.r3dg_raster_img_bytes(64, 48)
    elif flaw == "img-one-byte-short":
        a.img_bytes -= 1
    elif flaw == "no-depth2":
        a.out_depth2 = None
    elif flaw == "no-median":
        a.out_median_depth = None
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001, flaw


@pytest.mark.parametrize("flaw", ["img-of-the-default-layout", "no-depth2-cotangent", "no-median-cotangent",
                                  "cotangent-without-flag", "several-views-img-of-one"])
def test_backward_refusals(flaw):
    lib = _lib.load()
    a = _bwd_args(lib)
    if flaw == "img-of-the-default-layout":
        a.img_bytes = lib.r3dg_raster_img_bytes(64, 48)
    elif flaw == "no-depth2-cotangent":
        a.dL_dout_depth2 = None
    elif flaw == "no-median-cotangent":
        a.dL_dout_median_depth = None
    elif flaw == "cotangent-without-flag":
        a.depth_stats = 0
        a.img_bytes = lib.r3dg_raster_img_bytes(64, 48)
    elif flaw == "several-views-img-of-one":
        cams = (ctypes.c_float * 8)()
        a.V, a.view_cams = 2, ctypes.cast(cams, ctypes.c_void_p)
        a.geom_bytes = lib.r3dg_raster_views_geom_bytes(100, 5, 2)
    assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001, flaw


def test_fields_sit_with_the_other_mode_flags():
    fwd = [f[0] for f in _lib.RasterFwdArgs._fields_]
    bwd = [f[0] for f in _lib.RasterBwdArgs._fields_]
    assert fwd[-8:-5] == ["depth_stats", "out_depth2", "out_median_depth"] and fwd[-5] == "ray_depth"
    assert bwd[-9:-6] == ["depth_stats", "dL_dout_depth2", "dL_dout_median_depth"] and bwd[-6] == "ray_depth"


def test_keyword_defaults_are_off():
    for fn in (R.rasterize_gaussians, R.rasterize_views):
        assert inspect.signature(fn).parameters["depth_stats"].default is False, fn.__name__
    assert inspect.signature(R.GaussianRasterizer.__init__).parameters["depth_stats"].default is False
    for fn in (_C_raster.rasterize_gaussians, _C_raster.rasterize_gaussians_backward, _C_raster.rasterize_views,
               _C_raster.rasterize_views_backward):
        assert inspect.signature(fn).parameters["depth_stats"].default is None, fn.__name__
    assert not hasattr(R, "set_depth_stats") and not hasattr(_C_raster, "set_depth_stats")   # no process default


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
def test_host_layer_passes_the_flag_to_the_forward(monkeypatch, on):
    seen = []

    def fake(*args, **kw):
        seen.append(kw)
        raise _Stop()
    monkeypatch.setattr(R._C, "rasterize_gaussians", fake)
    monkeypatch.setattr(R._C, "rasterize_views", fake)
    rs, lv = _settings()
    P = lv["means3D"].shape[0]
    kw = {"depth_stats": True} if on else {}
    with pytest.raises(_Stop):
        R.GaussianRasterizer(rs, **kw)(means3D=lv["means3D"], means2D=torch.zeros(P, 3), opacities=lv["opacities"],
                                       shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"])
    with pytest.raises(_Stop):
        R.rasterize_views(lv["means3D"], torch.zeros(2, P, 3), lv["opacities"], settings=[rs, rs], shs=lv["shs"],
                          scales=lv["scales"], rotations=lv["rotations"], **kw)
    assert [k.get("depth_stats") for k in seen] == ([True, True] if on else [None, None])


def _render(rs, lv, geometry=True, **kw):
    """A one-view forward with means3D (geometry) or only shs (appearance) requiring grad; returns its outputs."""
    P = lv["means3D"].shape[0]
    return R.GaussianRasterizer(rs, **kw)(means3D=lv["means3D"].requires_grad_(geometry), means2D=torch.zeros(P, 3),
                                          opacities=lv["opacities"], shs=lv["shs"].requires_grad_(True),
                                          scales=lv["scales"], rotations=lv["rotations"])


@pytest.mark.parametrize("geometry", [True, False])
def test_library_backward_gets_the_flag_and_the_cotangents(monkeypatch, geometry):
    calls = fake_raster_library(monkeypatch)
    rs, lv = _settings()
    out = _render(rs, lv, geometry, depth_stats=True)
    g2, gm = torch.ones(1, 4, 5), torch.full((1, 4, 5), 2.0)
    torch.autograd.backward([out[10], out[11]], [g2, gm])
    name, kw = calls[-1]
    assert name == "rasterize_gaussians_backward" and kw["depth_stats"] is True
    assert kw["dL_dout_depth2"] is g2 and kw["dL_dout_median_depth"] is gm
    assert kw.get("geometry", True) is geometry
    # flag off: the call is exactly the flag-off call
    calls.clear()
    _render(rs, lv, geometry)[2].sum().backward()
    assert "depth_stats" not in calls[-1][1] and "dL_dout_depth2" not in calls[-1][1]


def test_deferred_count_rerun_through_backward_keeps_the_flag(monkeypatch):
    """The deferred-count repair re-runs the forward with the flag and differentiates the re-run's buffers."""
    calls = fake_raster_library(monkeypatch, overflow=True)
    rs, lv = _settings()
    R.set_deferred_count(True)
    try:
        out = _render(rs, lv, depth_stats=True)
    finally:
        R.set_deferred_count(False)
    with pytest.warns(UserWarning):
        out[10].sum().backward()
    assert [n for n, _ in calls] == ["rasterize_gaussians", "rasterize_gaussians_backward", "rasterize_gaussians",
                                     "rasterize_gaussians_backward"]
    assert calls[0][1]["_defer"] is True and "_defer" not in calls[2][1]
    assert calls[2][1].get("depth_stats") is True
    assert calls[3][1]["depth_stats"] is True and calls[3][1]["dL_dout_median_depth"] is None


def test_debug_snapshot_records_the_flag(monkeypatch, tmp_path):
    def fake(*args, **kw):
        raise _Stop()
    monkeypatch.setattr(R._C, "rasterize_gaussians", fake)
    monkeypatch.chdir(tmp_path)
    rs, lv = _settings(debug=True)
    P = lv["means3D"].shape[0]
    with pytest.raises(_Stop):
        R.rasterize_gaussians(lv["means3D"], torch.zeros(P, 3), torch.zeros(P, 0), lv["shs"], torch.Tensor([]),
                              lv["opacities"], lv["scales"], lv["rotations"], torch.Tensor([]), rs, depth_stats=True)
    saved = torch.load(tmp_path / "snapshot_fw.dump", weights_only=False)
    assert saved[-1]["depth_stats"] is True
