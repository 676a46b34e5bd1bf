"""Mip-Splatting's 3D filter without a GPU: the fp64 oracle (tests/filter3d_oracle.py) against autograd, central
differences and Mip-Splatting's determinant form; mass conservation; the f = 0 identities of filter3d.fold; and every
refusal of the host layer and the C ABI, none of which reaches the device."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import filter3d_oracle as fo
from relightable3dgaussian_b200 import _C_raster, _lib, filter3d
from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings, rasterize_gaussians

FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued


def _scales(n=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    s = torch.exp(torch.randn(n, 3, generator=g, dtype=torch.float64) * 2 - 4)
    f = torch.exp(torch.randn(n, generator=g, dtype=torch.float64) - 4)
    o = torch.rand(n, generator=g, dtype=torch.float64)
    return s, o, f


def test_per_axis_coef_equals_determinant_form():
    s, _, f = _scales()
    _, _, coef = fo.dilate(s, torch.ones(len(s), dtype=torch.float64), f)
    assert torch.allclose(coef, fo.coef_det(s, f), rtol=1e-13, atol=0)


def test_per_axis_coef_does_not_underflow_where_the_determinant_does():
    s = torch.full((1, 3), 1e-7, dtype=torch.float32)
    f = torch.tensor([1e-7])
    assert float((s.double() ** 2).prod()) < 1e-40                      # det1 ~ 1e-42 is subnormal in fp32
    assert float(torch.prod(s * s, 1)) < 2.0 ** -126                   # ... and loses its bits there
    _, o2 = filter3d.fold(s, torch.ones(1, 1), f)
    assert abs(float(o2) - 2 ** -1.5) < 1e-6                            # (1/2)^(3/2) per axis


def test_dcoef_matches_autograd_and_central_differences():
    s, o, f = _scales()
    s = torch.cat([s, torch.tensor([[0.0, 0.01, 0.02]], dtype=torch.float64)])       # s_k = 0 included
    f = torch.cat([f, torch.tensor([0.005], dtype=torch.float64)])
    o = torch.cat([o, torch.tensor([0.5], dtype=torch.float64)])
    x = s.clone().requires_grad_(True)
    coef = fo.dilate(x, torch.ones(len(s), dtype=torch.float64), f)[2]
    (g,) = torch.autograd.grad(coef.sum(), x)
    d = fo.dcoef(s, f)
    rows = (s != 0).all(1)
    # autograd forms g / s'^3 as 1 / s' - s^2 / s'^3, which cancels where s >> f: 2e-11 relative on these rows
    assert torch.allclose(d[rows], g[rows], rtol=1e-9, atol=0)
    h = 1e-7 * s.abs().clamp_min(1e-4)
    for k in range(3):
        e = torch.zeros_like(s)
        e[:, k] = h[:, k]
        fd = (fo.dilate(s + e, o, f)[2] - fo.dilate(s - e, o, f)[2]) / (2 * h[:, k])
        ok = (s[:, k] != 0)
        # (central differences of coef, which is ~1 where s >> f, carry ~1e-16 / h of cancellation)
        assert torch.allclose(d[ok, k], fd[ok], rtol=1e-4, atol=1e-7 * float(d[:, k].abs().max())), k
    # s_k = 0: coef is |s_k| (...) — the one-sided slope from above is the form's value, which is finite
    z = s.shape[0] - 1
    up = (fo.dilate(s[z:] + torch.tensor([[1e-9, 0, 0]], dtype=torch.float64), o[z:], f[z:])[2]
          - fo.dilate(s[z:], o[z:], f[z:])[2]) / 1e-9
    assert torch.isfinite(d[z]).all() and abs(float(up) - float(d[z, 0])) <= 1e-4 * abs(float(d[z, 0]))


def test_mass_is_conserved():
    s, o, f = _scales()
    sp, op, _ = fo.dilate(s, o, f)
    assert torch.allclose(op * sp.prod(1), o * s.prod(1), rtol=1e-13, atol=0)


def test_fold_matches_the_oracle_and_is_the_identity_for_f_zero():
    s, o, f = _scales(256, 3)
    s32, o32, f32 = s.float(), o.float()[:, None], f.float()[:, None]
    sp, op = filter3d.fold(s32, o32, f32)
    sp64, op64, _ = fo.dilate(s32.double(), o32.double(), f32.double())
    assert torch.allclose(sp.double(), sp64, rtol=4 * fo.EPS32, atol=0)
    assert torch.allclose(op.double()[:, 0], op64, rtol=16 * fo.EPS32, atol=0)
    # f = 0: |s| and o exactly, for s = 0, negative s and every s whose square is a normal float
    s0 = torch.cat([s32, -s32[:8], torch.zeros(1, 3), torch.tensor([[2.0 ** -63, 1.0, 2.0 ** 63]])])
    o0 = torch.rand(len(s0), 1)
    sp0, op0 = filter3d.fold(s0, o0, torch.zeros(len(s0)))
    assert torch.equal(sp0, s0.abs()) and torch.equal(op0, o0)
    assert torch.equal(fo.dcoef(s0.double(), torch.zeros(len(s0), dtype=torch.float64)), torch.zeros(len(s0), 3,
                                                                                                     dtype=torch.float64))


def test_chain_rule_oracle_against_autograd():
    s, o, f = _scales(32, 5)
    g = torch.Generator().manual_seed(9)
    g_sp, g_op = torch.randn(32, 3, generator=g, dtype=torch.float64), torch.randn(32, generator=g, dtype=torch.float64)
    x, y = s.clone().requires_grad_(True), o.clone().requires_grad_(True)
    sp, op, _ = fo.dilate(x, y, f)
    gx, gy = torch.autograd.grad((sp * g_sp).sum() + (op * g_op).sum(), (x, y))
    ds, do, _ = fo.chain(s, o, f, g_sp, g_op)
    assert torch.allclose(ds, gx, rtol=1e-12, atol=0) and torch.allclose(do, gy, rtol=1e-12, atol=0)


def test_compute_oracle_principal_point_and_fallbacks():
    # one camera looking down +z from the origin; FoV intrinsics put the principal point at the centre
    views = torch.eye(4, dtype=torch.float64).reshape(1, 16)
    intr = torch.tensor([[100.0, 100.0, 32.0, 24.0, 64.0, 48.0]], dtype=torch.float64)
    means = torch.tensor([[0.0, 0.0, 2.0], [0.0, 0.0, -1.0], [0.0, 0.0, 4.0]], dtype=torch.float64)
    f, seen, _, _ = fo.compute(means, views, intr, 100.0)
    assert seen.tolist() == [True, False, True]
    assert torch.allclose(f, torch.tensor([2.0, 4.0, 4.0], dtype=torch.float64) / 100 * 0.2 ** 0.5)   # unseen: max d
    f0, _, _, _ = fo.compute(means[1:2], views, intr, 100.0)
    assert torch.equal(f0, torch.zeros(1, dtype=torch.float64))


def test_intrinsics_from_camera_attributes():
    fov = SimpleNamespace(image_width=64, image_height=48, FoVx=1.0, FoVy=0.8, fx=None)
    fx = np.float32(64 / (2 * np.tan(0.5)))
    assert filter3d._intrinsics(fov) == (float(fx), float(np.float32(48 / (2 * np.tan(0.4)))), 32.0, 24.0)
    real = SimpleNamespace(image_width=64, image_height=48, fx=50.5, fy=51.25, cx=30.0, cy=20.0)
    assert filter3d._intrinsics(real) == (50.5, 51.25, 30.0, 20.0)


# ---- refusals ------------------------------------------------------------------------------------------------------

def test_check_filter_3d_refusals():
    P = 10
    with pytest.raises(ValueError, match="shape"):
        _C_raster._check_filter_3d(torch.zeros(P + 1), P, None)
    with pytest.raises(ValueError, match="shape"):
        _C_raster._check_filter_3d(torch.zeros(P, 2), P, None)
    with pytest.raises(ValueError, match="CUDA"):
        _C_raster._check_filter_3d(torch.zeros(P), P, None)
    with pytest.raises(ValueError, match="CUDA"):
        _C_raster._check_filter_3d(torch.zeros(P, 1), P, torch.empty(0))
    with pytest.raises(ValueError, match="cov3D_precomp"):
        _C_raster._check_filter_3d(torch.zeros(P), P, torch.zeros(P, 6))
    with pytest.raises(ValueError, match="tensor"):
        _C_raster._check_filter_3d([0.0] * P, P, None)
    assert _C_raster._check_filter_3d(None, P, torch.zeros(P, 6)) is None


def test_rasterize_gaussians_refuses_before_any_launch():
    P = 4
    rs = GaussianRasterizationSettings(8, 8, 1.0, 1.0, 4.0, 4.0, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0,
                                       torch.zeros(3), False, False, False, False)
    args = (torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 0), torch.zeros(P, 1, 3), torch.empty(0),
            torch.ones(P, 1), torch.ones(P, 3), torch.zeros(P, 4), torch.empty(0), rs)
    for bad in (torch.zeros(P + 1), torch.zeros(P, 2), torch.zeros(P), torch.zeros(P, dtype=torch.float64)):
        with pytest.raises(ValueError):
            rasterize_gaussians(*args, filter_3d=bad)


def test_requires_grad_and_dtype_are_refused_on_the_device_check_path(monkeypatch):
    class FakeCuda(torch.Tensor):
        @property
        def is_cuda(self):
            return True
    P = 3
    t = torch.zeros(P).as_subclass(FakeCuda)
    assert _C_raster._check_filter_3d(t, P, None) is t
    with pytest.raises(ValueError, match="float32"):
        _C_raster._check_filter_3d(torch.zeros(P, dtype=torch.float64).as_subclass(FakeCuda), P, None)
    with pytest.raises(ValueError, match="contiguous"):
        _C_raster._check_filter_3d(torch.zeros(P, 2)[:, 0].as_subclass(FakeCuda), P, None)
    with pytest.raises(ValueError, match="grad"):
        _C_raster._check_filter_3d(torch.zeros(P).as_subclass(FakeCuda).requires_grad_(True), P, None)


def test_c_abi_refusals():
    lib = _lib.load()
    a = _lib.RasterFwdArgs()
    a.P, a.S, a.W, a.H = 10, 0, 16, 16
    a.colors_precomp = a.cov3D_precomp = a.filter_3d = FAKE
    assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001
    assert _lib.RasterFwdArgs().filter_3d is None and _lib.RasterBwdArgs().filter_3d is None    # zeroed: off
    for flaw in ("cov3D", "no-opacities"):
        b = _lib.RasterBwdArgs()
        b.P, b.S, b.W, b.H = 10, 0, 16, 16
        for n in ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dscales", "dL_drotations"):
            setattr(b, n, FAKE)
        b.filter_3d = FAKE
        if flaw == "cov3D":
            b.cov3D_precomp = b.opacities = FAKE
        assert lib.r3dg_raster_backward(ctypes.byref(b), None) == -10001, flaw
    # the filter kernel: bad P, F, V and missing pointers are refused; P = 0 is a no-op
    call = lambda P, V, F, ptrs=(FAKE, FAKE, FAKE), out=FAKE, tmp=FAKE, nb=256: lib.r3dg_filter3d_compute(
        P, V, *ptrs, ctypes.c_float(F), out, tmp, nb, None)
    assert call(0, 0, 1.0, (None, None, None), None, None, 0) == 0
    assert call(-1, 1, 1.0) == -10001
    assert call(5, 0, 1.0) == -10001
    for F in (0.0, -1.0, float("inf"), float("nan")):
        assert call(5, 1, F) == -10001
    assert call(5, 1, 1.0, (None, FAKE, FAKE)) == -10001
    assert call(5, 1, 1.0, nb=lib.r3dg_filter3d_tmp_bytes(5) - 1) == -10001
    assert call(5, 1, 1.0, tmp=None) == -10001


def test_compute_3d_filter_refuses_on_the_host():
    with pytest.raises(ValueError, match="camera"):
        filter3d.compute_3d_filter(torch.zeros(3, 3), [])
    cam = SimpleNamespace(image_width=4, image_height=4, fx=1.0, fy=1.0, cx=2.0, cy=2.0, world_view_transform=torch.eye(4))
    with pytest.raises(ValueError, match="CUDA"):
        filter3d.compute_3d_filter(torch.zeros(3, 3), [cam])
    with pytest.raises(ValueError, match=r"\[P,3\]"):
        filter3d.compute_3d_filter(torch.zeros(3, 2), [cam])
