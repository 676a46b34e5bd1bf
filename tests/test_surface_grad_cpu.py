"""Pseudo-normal / surface-xyz gradients without a GPU: the workspace size, the C layer's refusals before any launch,
the Python refusal without the pseudo-normal pass, and the fp64 restatement used as truth on the GPU against the CPU
oracle of the forward."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import rel_l2
from oracle import oracle
from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200 import rasterizer as R
from surface_oracle import surface_normal

FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued


def _bwd_args(lib, P=100, S=5, W=64, H=48, V=1):
    a = _lib.RasterBwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_views_geom_bytes(P, S, V)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_views_img_bytes(W, H, V)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.dL_dout_color = a.dL_dout_opacity = a.dL_dout_depth = a.dL_dout_feature = FAKE
    return a


def test_surface_grad_bytes_exact():
    """The combined depth and opacity planes [2,V,H,W] and the camera partials [V,9,blocks of 32x8 pixels], each
    rounded up to 256 bytes; W, H and V below 1 are sized as 1."""
    lib = _lib.load()
    up = lambda n: -(-n // 256) * 256
    for W, H, V in [(1, 1, 1), (0, -3, 0), (2, 2, 1), (33, 9, 1), (64, 48, 3), (800, 800, 1), (1600, 1200, 16),
                    (37, 2, 5), (1, 37, 64)]:
        w, h, v = max(W, 1), max(H, 1), max(V, 1)
        blocks = -(-w // 32) * -(-h // 8)
        want = up(8 * v * w * h) + up(36 * v * blocks)
        assert lib.r3dg_raster_surface_grad_bytes(W, H, V) == want, (W, H, V)
    assert lib.r3dg_raster_surface_grad_bytes(800, 800, 1) == 5120000 + 90112


def test_camera_grad_bytes_unchanged():
    assert _lib.load().r3dg_raster_cam_grad_bytes(10**6, 8) == 8750592


@pytest.mark.parametrize("P", [100, 0])
@pytest.mark.parametrize("V", [1, 3])
def test_surface_refusals(P, V):
    lib = _lib.load()
    W, H = 64, 48
    need = lib.r3dg_raster_surface_grad_bytes(W, H, V)
    cams = (ctypes.c_float * (4 * V))(*([1.0, 1.0, 32.0, 24.0] * V))

    def args(**kw):
        a = _bwd_args(lib, P=P, W=W, H=H, V=V)
        if V > 1:
            a.V, a.view_cams = V, ctypes.cast(cams, ctypes.c_void_p)
        a.fwd_opacity = a.fwd_depth = FAKE
        a.surface_work, a.surface_work_bytes = FAKE, need
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    cases = [dict(dL_dout_normal=FAKE, fwd_opacity=None), dict(dL_dout_normal=FAKE, fwd_depth=None),
             dict(dL_dout_surface_xyz=FAKE, fwd_opacity=None), dict(dL_dout_surface_xyz=FAKE, fwd_depth=None),
             dict(dL_dout_normal=FAKE, dL_dout_surface_xyz=FAKE, fwd_opacity=None, fwd_depth=None),
             dict(dL_dout_normal=FAKE, surface_work=None), dict(dL_dout_surface_xyz=FAKE, surface_work_bytes=need - 1),
             dict(dL_dout_normal=FAKE, dL_dout_surface_xyz=FAKE, surface_work_bytes=0),
             dict(dL_dout_normal=FAKE, dL_dout_depth=None), dict(dL_dout_surface_xyz=FAKE, dL_dout_opacity=None)]
    for kw in cases:
        assert lib.r3dg_raster_backward(ctypes.byref(args(**kw)), None) == -10001, kw


def test_one_view_surface_backward_needs_the_principal_point():
    """A one-view library call reads cx, cy from the argument struct: the host layer refuses to leave them unset."""
    from relightable3dgaussian_b200 import _C_raster
    t = torch.zeros(1)
    with pytest.raises(ValueError, match="principal point"):
        _C_raster._surface_args(_lib.RasterBwdArgs(), (t, None, t, t), 4, 4, 1, "cpu")
    assert _C_raster._surface_args(_lib.RasterBwdArgs(), (None, None, t, t), 4, 4, 1, "cpu") is None


def _settings(pseudo_normal):
    return R.GaussianRasterizationSettings(4, 5, 1.0, 1.0, 2.0, 1.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 3,
                                           torch.zeros(3), False, True, pseudo_normal, False)


def test_surface_grads_without_pseudo_normal_is_refused(monkeypatch):
    called = []
    monkeypatch.setattr(R._C, "rasterize_gaussians", lambda *a, **k: called.append(1))
    monkeypatch.setattr(R._C, "rasterize_views", lambda *a, **k: called.append(1))
    P = 7
    leaves = dict(means3D=torch.randn(P, 3), opacities=torch.rand(P, 1), shs=torch.randn(P, 16, 3),
                  scales=torch.rand(P, 3), rotations=torch.randn(P, 4))
    rs = _settings(False)
    with pytest.raises(ValueError, match="computer_pseudo_normal"):
        R.GaussianRasterizer(rs, surface_grads=True)(means2D=torch.zeros(P, 3), **leaves)
    with pytest.raises(ValueError, match="computer_pseudo_normal"):
        R.rasterize_gaussians(leaves["means3D"], torch.zeros(P, 3), torch.empty(P, 0), leaves["shs"], torch.Tensor([]),
                              leaves["opacities"], leaves["scales"], leaves["rotations"], torch.Tensor([]), rs,
                              surface_grads=True)
    with pytest.raises(ValueError, match="computer_pseudo_normal"):
        R.rasterize_views(leaves["means3D"], torch.zeros(2, P, 3), leaves["opacities"], settings=[rs, rs],
                          shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"], surface_grads=True)
    assert not called
    assert R.GaussianRasterizer(_settings(True)).surface_grads is False
    assert len(R.GaussianRasterizationSettings._fields) == 16


def _images(W, H, seed):
    """Rendered-like opacity and depth: opacity in (0, 1] with exact-zero background pixels (depth 0 there too),
    depth = opacity * z with a smooth z plus noise."""
    g = np.random.default_rng(seed)
    o = g.uniform(0.05, 1.0, (H, W)).astype(np.float32)
    o[g.random((H, W)) < 0.15] = 0.0
    yy, xx = np.mgrid[0:H, 0:W]
    z = 3.0 + 0.5 * np.sin(xx / 7.0) + 0.3 * np.cos(yy / 5.0) + 0.05 * g.standard_normal((H, W))
    d = (o * z).astype(np.float32)
    return o[None], d[None]


@pytest.mark.parametrize("W,H", [(37, 29), (64, 48), (1, 1), (1, 7), (9, 1), (2, 2), (2, 13), (31, 2), (33, 9)])
def test_fp64_restatement_matches_oracle(W, H):
    """The truth of the GPU tests is the forward itself: on random images (borders, zero-opacity pixels, 1-2 pixel
    wide images) it matches the CPU oracle of surface_normal_kernel up to fp32 rounding."""
    o, d = _images(W, H, seed=W * 100 + H)
    rng = np.random.default_rng(7)
    Q = np.linalg.qr(rng.standard_normal((3, 3)))[0]
    V = np.eye(4, dtype=np.float32)
    V[:3, :3] = Q
    V[3, :3] = rng.standard_normal(3)
    tfx, tfy, cx, cy = 0.6, 0.45, W / 2.0 + 0.3, H / 2.0 - 0.2
    want_n, want_x = oracle.surface_normal(o, d, V, W, H, tfx, tfy, cx, cy)
    got_n, got_x = surface_normal(torch.from_numpy(o).double(), torch.from_numpy(d).double(),
                                  torch.from_numpy(V).double(), W, H, tfx, tfy, cx, cy)
    got_n, got_x = got_n.numpy(), got_x.numpy()
    assert np.isfinite(got_n).all() and np.isfinite(got_x).all()
    assert rel_l2(got_x, want_x) <= 1e-6
    np.testing.assert_allclose(got_x, want_x, rtol=1e-6, atol=1e-6)
    if W == 1 or H == 1:
        # one stencil direction vanishes: n = 0 exactly, so no normal.  (The fp32 forward's vertical stencil of a
        # one-row image is rounding noise of its FMA chain rather than 0, so its normals there are not compared.)
        assert (got_n == 0).all()
        return
    zero = (want_n == 0).all(0)
    assert ((got_n == 0).all(0) == zero).all()             # the same pixels get no normal
    assert not zero.all()
    # the normal is a unit vector (rotated by an orthogonal M) wherever it exists
    np.testing.assert_allclose(np.linalg.norm(got_n[:, ~zero], axis=0), 1.0, atol=1e-12)
    np.testing.assert_allclose(got_n, want_n, atol=2e-4)
    assert rel_l2(got_n, want_n) <= 1e-5
