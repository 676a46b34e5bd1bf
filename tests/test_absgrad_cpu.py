"""Absolute screen-space gradients (absgrad) without a GPU: the fp64 oracle (absgrad64.py) against an independent
per-pixel autograd and its invariants, the C layer's plumbing and refusals, the host keywords and the process
defaults (rasterizer.set_absgrad, densify.install)."""
import ctypes
import inspect

import pytest
import torch

import absgrad64
import raster64
import densify_oracle as do
from helpers import fake_raster_library
from relightable3dgaussian_b200 import _C_raster, _lib, densify
from relightable3dgaussian_b200 import rasterizer as R

FAKE = 256               # a non-NULL device pointer the library never dereferences (refused before any launch)
W = H = 16


def _scene(seed=0, P=6, tiny=None):
    """A one-tile scene in the forward state raster64.Walk reads, list order = depth order.  `tiny` = (x, y): one more
    Gaussian, last in the list, of 0.25 px standard deviation 0.2 px off the centre of that pixel, so that only that
    pixel composites it."""
    g = torch.Generator().manual_seed(seed)
    m = 2.0 + 12.0 * torch.rand(P, 2, generator=g, dtype=torch.float64)
    s = 1.0 + 2.0 * torch.rand(P, 2, generator=g, dtype=torch.float64)
    th = 3.14 * torch.rand(P, generator=g, dtype=torch.float64)
    c, si = torch.cos(th), torch.sin(th)
    R2 = torch.stack([torch.stack([c, -si], -1), torch.stack([si, c], -1)], -2)
    cov = R2 @ torch.diag_embed(s ** 2) @ R2.transpose(1, 2)
    inv = torch.linalg.inv(cov)
    op = 0.3 + 0.5 * torch.rand(P, generator=g, dtype=torch.float64)
    co = torch.stack([inv[:, 0, 0], inv[:, 0, 1], inv[:, 1, 1], op], 1)
    if tiny is not None:
        m = torch.cat([m, torch.tensor([[tiny[0] + 0.2, tiny[1] - 0.1]], dtype=torch.float64)])
        co = torch.cat([co, torch.tensor([[16.0, 0.0, 16.0, 0.5]], dtype=torch.float64)])
        P += 1
    S = 2
    st = dict(point_list=torch.arange(P), ranges=torch.tensor([[0, P]]),
              n_contrib=torch.full((H, W), P, dtype=torch.int32), means2D=m, conic_opacity=co,
              rgb=torch.rand(P, 3, generator=g, dtype=torch.float64),
              depths=1.0 + torch.rand(P, generator=g, dtype=torch.float64),
              features=torch.rand(P, S, generator=g, dtype=torch.float64))
    cots = [torch.randn(c, H, W, generator=g, dtype=torch.float64) for c in (3, 1, 1, S)]
    bg = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64)
    return st, cots, bg, S


def _per_pixel_autograd(st, cots, bg, S):
    """sum over pixels of |d(pixel's loss) / d mean2D| by fp64 autograd of every pixel's own composite, with the pairs'
    accept decisions of the Walk held fixed, in the kernel's units (0.5 W, 0.5 H per pixel)."""
    wk = raster64.Walk(st, [0], W, H)
    planes = torch.cat([c.reshape(c.shape[0], -1) for c in cots], 0)[:, wk.pix].T

    def losses(m2):
        dx = m2[wk.ids][..., 0] - wk.px.double()[:, None]
        dy = m2[wk.ids][..., 1] - wk.py.double()[:, None]
        power = -0.5 * (wk.ca * dx ** 2 + wk.cc * dy ** 2) - wk.cb * dx * dy
        alpha = torch.where(wk.valid, wk.op * torch.exp(power.clamp_max(0.0)), torch.zeros_like(power))
        return (wk.composite(st, bg, S, alpha) * planes).sum(1)
    J = torch.autograd.functional.jacobian(losses, st["means2D"].clone())              # [n, P, 2]
    return (J.abs() * torch.tensor([0.5 * W, 0.5 * H], dtype=torch.float64)).sum(0)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_matches_per_pixel_autograd(seed):
    st, cots, bg, S = _scene(seed)
    absg, sig = absgrad64.row_truth(st, raster64.walks_of(st, W, H), cots, bg, W, H, S)
    want = _per_pixel_autograd(st, cots, bg, S)
    assert torch.allclose(absg, want, rtol=1e-10, atol=1e-12), (absg, want)
    # the signed sums are raster64's dL_dmeans2D
    g64, _ = raster64.row_truth(st, raster64.walks_of(st, W, H), cots, bg, W, H, S)["dL_dmeans2D"]
    assert torch.allclose(sig, g64, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_invariants(seed):
    st, cots, bg, S = _scene(seed, tiny=(7, 9))
    walks = raster64.walks_of(st, W, H)
    absg, sig = absgrad64.row_truth(st, walks, cots, bg, W, H, S)
    assert bool((absg >= sig.abs() * (1 - 1e-12)).all())
    # the large Gaussians cover many pixels pulling in different directions: strictly more than the signed sum
    assert bool((absg[:-1] > sig[:-1].abs() * (1 + 1e-6)).any())
    # the tiny one: one pixel composites it, so nothing cancels
    pix = walks[0].valid[:, -1].nonzero()[:, 0]
    assert pix.numel() == 1 and int(walks[0].pix[pix]) == 9 * W + 7
    assert torch.allclose(absg[-1], sig[-1].abs(), rtol=1e-14, atol=0) and bool((absg[-1] > 0).all())


def test_abi_field_and_workspace():
    lib = _lib.load()
    names = [f[0] for f in _lib.RasterBwdArgs._fields_]
    assert names.index("dL_dmeans2D_abs") == names.index("antialiasing") - 1
    assert _lib.RasterBwdArgs().dL_dmeans2D_abs is None                     # zero-initialised: NULL, the old call
    # the gradient rows' workspace is unchanged; absgrad's two accumulators per row come on top
    assert lib.r3dg_raster_bwd_det_bytes(1000, 5) == 384_000 + 4096
    assert lib.r3dg_raster_bwd_det_absgrad_bytes(1000) == 48_128 + 512     # 24 B per accumulator, 2 flag bits
    assert lib.r3dg_raster_bwd_det_absgrad_bytes(0) == lib.r3dg_raster_bwd_det_absgrad_bytes(1) > 0


def _bwd_args(lib, P=100, S=5, Wd=64, Hd=48):
    a = _lib.RasterBwdArgs()
    a.P, a.S, a.W, a.H = P, S, Wd, Hd
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(Wd, Hd)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.dL_dmeans2D = a.dL_dopacity = a.dL_dmeans3D = a.dL_dcov3D = a.dL_dscales = a.dL_drotations = FAKE
    a.dL_dmeans2D_abs = FAKE
    return a


@pytest.mark.parametrize("flaw", ["det-rows-only-work", "det-one-byte-short", "partial-geometry"])
def test_backward_refusals_with_absgrad(flaw):
    lib = _lib.load()
    a = _bwd_args(lib)
    rows = lib.r3dg_raster_bwd_det_bytes(100, 5)
    if flaw.startswith("det"):
        a.deterministic, a.det_work = 1, FAKE
        a.det_work_bytes = rows if flaw == "det-rows-only-work" else rows + lib.r3dg_raster_bwd_det_absgrad_bytes(100) - 1
    elif flaw == "partial-geometry":
        a.dL_dcov3D = None
    assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001, flaw


@pytest.mark.parametrize("fn", [R.GaussianRasterizer.__init__, R.rasterize_gaussians, R.rasterize_views,
                                _C_raster.rasterize_gaussians_backward, _C_raster.rasterize_views_backward])
def test_keyword_defaults_off(fn):
    assert inspect.signature(fn).parameters["absgrad"].default is False


def _settings():
    rs = R.GaussianRasterizationSettings(4, 5, 1.0, 1.0, 2.5, 2.0, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3,
                                         torch.zeros(3), False, True, True, False)
    g = torch.Generator().manual_seed(0)
    lv = dict(means3D=torch.randn(7, 3, generator=g), opacities=torch.rand(7, 1, generator=g),
              shs=torch.randn(7, 16, 3, generator=g), scales=torch.rand(7, 3, generator=g),
              rotations=torch.randn(7, 4, generator=g))
    return rs, lv


def _backward_kw(calls):
    return [kw for name, kw in calls if name.endswith("backward")]


def _render_one(rs, lv, means2D, **kw):
    out = R.GaussianRasterizer(rs, **kw)(means3D=lv["means3D"], means2D=means2D, opacities=lv["opacities"],
                                         shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"])
    out[2].sum().backward()


@pytest.mark.parametrize("how", ["off", "keyword", "process-default"])
def test_calls_take_the_mode(monkeypatch, how):
    """The autograd node gets the call's absgrad mode, the keyword or set_absgrad's process default, and hands it to
    the library backward of one view and of V views."""
    calls = fake_raster_library(monkeypatch)
    rs, lv = _settings()
    R.set_absgrad(how == "process-default")
    try:
        kw = {"absgrad": True} if how == "keyword" else {}
        _render_one(rs, lv, torch.zeros(7, 3, requires_grad=True), **kw)
        out = R.rasterize_views(lv["means3D"], torch.zeros(2, 7, 3, requires_grad=True), lv["opacities"],
                                settings=[rs, rs], shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"], **kw)
        out[2].sum().backward()
    finally:
        R.set_absgrad(False)
    assert [k.get("absgrad") for k in _backward_kw(calls)] == [True if how != "off" else None] * 2


@pytest.mark.parametrize("absgrad, means2d, geometry, want", [
    (False, True, True, {}), (True, True, True, {"absgrad": True}),
    (True, False, True, {}),          # means2D needs no gradient: nothing computed, nothing set
    (True, False, False, {})])        # (the appearance-only backward has no geometry half)
def test_backward_asks_for_absgrad_only_when_means2d_needs_a_gradient(monkeypatch, absgrad, means2d, geometry, want):
    calls = fake_raster_library(monkeypatch)
    rs, lv = _settings()
    lv["means3D"].requires_grad_(geometry)
    lv["shs"].requires_grad_(True)
    means2D = torch.zeros(7, 3, requires_grad=means2d)
    _render_one(rs, lv, means2D, absgrad=absgrad)
    (kw,) = _backward_kw(calls)
    assert {k: v for k, v in kw.items() if k == "absgrad"} == want
    assert kw.get("geometry", True) is geometry
    assert (getattr(means2D, "absgrad", None) is not None) == bool(want)


def test_attribute_accumulates_like_grad():
    t = torch.zeros(3, 3)
    R._set_absgrad(t, torch.ones(3, 2))
    R._set_absgrad(t, torch.full((3, 2), 2.0))
    assert torch.equal(t.absgrad, torch.full((3, 2), 3.0))


def test_set_absgrad_round_trips_through_the_backward(monkeypatch):
    calls = fake_raster_library(monkeypatch)
    rs, lv = _settings()
    assert R._ABSGRAD is False
    R.set_absgrad(True)
    try:
        _render_one(rs, lv, torch.zeros(7, 3, requires_grad=True))
    finally:
        R.set_absgrad(False)
    _render_one(rs, lv, torch.zeros(7, 3, requires_grad=True))
    _render_one(rs, lv, torch.zeros(7, 3, requires_grad=True), absgrad=True)
    assert [k.get("absgrad") for k in _backward_kw(calls)] == [True, None, True]


def _model():
    case = do.densify_case("s1_p7")
    return do.build_model(case, do.StandIn)


def test_densification_refuses_a_missing_or_misshaped_absgrad(monkeypatch):
    calls = []
    monkeypatch.setattr(_lib, "call", lambda *a, **k: calls.append(a))
    m = _model()
    P = m._xyz.shape[0]
    vpt = torch.zeros(P, 3)
    with pytest.raises(RuntimeError, match="absgrad"):
        densify.add_densification_stats(m, vpt, torch.ones(P, dtype=torch.bool), torch.ones(P, 1), absgrad=True)
    for shape in ((P, 3), (P + 1, 2), (2, P, 2), (P,)):
        vpt.absgrad = torch.zeros(shape)
        with pytest.raises(ValueError, match="absgrad"):
            densify.add_densification_stats(m, vpt, torch.ones(P, dtype=torch.bool), torch.ones(P, 1), absgrad=True)
    vpt.absgrad = torch.zeros(P, 2)            # the right shape, on the CPU: refused as every other CPU tensor is
    with pytest.raises(RuntimeError, match="CUDA"):
        densify.add_densification_stats(m, vpt, torch.ones(P, dtype=torch.bool), torch.ones(P, 1), absgrad=True)
    assert calls == []


@pytest.mark.parametrize("absgrad", [False, True])
def test_install_round_trip(monkeypatch, absgrad):
    seen = []
    monkeypatch.setattr(densify, "add_densification_stats", lambda *a, **k: seen.append(k))

    class M(do.StandIn):
        pass
    orig = M.add_densification_stats
    densify.install(M, absgrad=absgrad)
    try:
        M.add_densification_stats(_model(), None, None, None)
    finally:
        densify.uninstall()
    assert seen == [{"absgrad": absgrad}]
    assert M.add_densification_stats is orig
