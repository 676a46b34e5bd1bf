"""Smoothness regularisers without a GPU: the PyTorch restatement (tests/smooth_oracle.py) against the outputs and
autograd gradients of the reference's own function bodies (tests/golden/smooth.npz), argument checks of the C ABI,
install() / uninstall(), and the Python-level rejections."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

import smooth_oracle as so
from helpers import GOLDEN
from relightable3dgaussian_b200 import _lib

G = np.load(os.path.join(GOLDEN, "smooth.npz"))


def _pinned(name, got64, got32):
    """fp64 to 1e-12; fp32 to a few ulp (oneDNN picks its CPU convolution kernels by instruction set)."""
    for key, (v, grads) in (("64", got64), ("32", got32)):
        tol = 1e-12 if key == "64" else 1e-6
        ref = G[f"{name}/value{key}"]
        assert abs(float(v) - float(ref)) <= tol * max(abs(float(ref)), 1e-3), (name, key, float(v), float(ref))
        for gname, g in grads.items():
            ref = G[f"{name}/{gname}{key}"]
            assert g.shape == ref.shape, (name, gname)
            assert np.abs(g.numpy() - ref).max() <= tol * max(np.abs(ref).max(), 1e-3), (name, gname, key)


@pytest.mark.parametrize("case", so.EDGE_CASES, ids=[c[0] for c in so.EDGE_CASES])
def test_edge_aware_oracle_matches_reference_function_golden(case):
    name, kind, Cd, Ci, H, W, seed = case
    d, i, cot = so.smooth_case(kind, Cd, Ci, H, W, seed)
    got = []
    for dt in (torch.float64, torch.float32):
        v, (gd, gi) = so.value_and_grads(so.first_order_edge_aware_loss, [d, i], cot, dt)
        assert v.shape == ()
        got.append((v, {"grad_data": gd, "grad_img": gi}))
    _pinned(f"edge/{name}", *got)
    if kind == "constdata" or (H, W) == (1, 1):
        # exactly 0 in fp64.  In fp32 the reference's weighted tap sums (-a/8 - a/4 ...) round and need not cancel;
        # the kernels take differences of opposite taps first, so they give 0 there too (tests/test_smooth_gpu.py).
        for k in ("value", "grad_data", "grad_img"):
            assert not G[f"edge/{name}/{k}64"].any(), k


@pytest.mark.parametrize("case", so.TV_CASES, ids=[c[0] for c in so.TV_CASES])
def test_tv_oracle_matches_reference_function_golden(case):
    name, shape, permuted, seed = case
    x, cot = so.tv_case(shape, permuted, seed)
    assert x.is_contiguous() != permuted
    got = []
    for dt in (torch.float64, torch.float32):
        v, (gx,) = so.value_and_grads(so.tv_loss, [x], cot, dt)
        got.append((v, {"grad": gx}))
    _pinned(f"tv/{name}", *got)


def test_spatial_gradient_normalisation_and_padding():
    """Sobel / 8 with replicate padding: a ramp of slope 1 has response exactly 1 everywhere inside and 1/2 on the
    replicated border columns; the response is [B,C,2,H,W] with d/dx first."""
    x = torch.arange(6, dtype=torch.float64).view(1, 1, 1, 6).expand(1, 2, 4, 6)
    g = so.spatial_gradient(x)
    assert g.shape == (1, 2, 2, 4, 6)
    gx, gy = g[0, :, 0].abs(), g[0, :, 1]
    assert torch.equal(gx[..., 1:-1], torch.ones(2, 4, 4, dtype=torch.float64))
    assert torch.equal(gx[..., [0, -1]], torch.full((2, 4, 2), 0.5, dtype=torch.float64))
    assert not gy.any()


def test_abi_rejects_bad_arguments_before_launching():
    lib = _lib.load()
    n0 = lib.r3dg_launch_count()
    p = ctypes.c_void_p(256)                 # never dereferenced: every call below fails its checks first
    tmp = lib.r3dg_edge_aware_tmp_bytes(3, 3, 40, 50)
    assert tmp > 0 and tmp % 256 == 0 and lib.r3dg_edge_aware_tmp_bytes(3, 3, 400, 500) > tmp
    assert lib.r3dg_edge_aware_tmp_bytes(1, 3, 40, 50) == lib.r3dg_edge_aware_tmp_bytes(3, 1, 40, 50) == tmp
    for Cd, Ci, H, W in ((0, 3, 8, 8), (3, 0, 8, 8), (3, 3, 0, 8), (3, 3, 8, 0), (-1, 1, 8, 8), (2, 3, 8, 8), (3, 2, 8, 8)):
        assert lib.r3dg_edge_aware_tmp_bytes(Cd, Ci, H, W) == 0
        assert lib.r3dg_edge_aware_forward(Cd, Ci, H, W, p, p, p, p, 1 << 20, None) == -10001
        assert lib.r3dg_edge_aware_backward(Cd, Ci, H, W, p, p, p, p, p, None) == -10001
    for k in range(4):                         # a NULL in each pointer argument of the forward
        ptrs = [p] * 4
        ptrs[k] = None
        assert lib.r3dg_edge_aware_forward(3, 1, 40, 50, *ptrs, tmp, None) == -10001
    for k in range(3):                         # ... and in each input of the backward
        ptrs = [p] * 3
        ptrs[k] = None
        assert lib.r3dg_edge_aware_backward(3, 1, 40, 50, *ptrs, p, p, None) == -10001
    assert lib.r3dg_edge_aware_backward(3, 1, 40, 50, p, p, p, None, None, None) == -10001   # no output at all
    assert lib.r3dg_edge_aware_forward(3, 3, 40, 50, p, p, p, p, tmp - 1, None) == -10001
    assert lib.r3dg_edge_aware_forward(65536, 1, 8, 8, p, p, p, p, 1 << 30, None) == -10002
    assert lib.r3dg_edge_aware_backward(1, 1, 1 << 16, 1 << 15, p, p, p, p, p, None) == -10002

    tmp = lib.r3dg_tv_tmp_bytes(3, 40, 50)
    assert tmp > 0 and tmp % 256 == 0 and lib.r3dg_tv_tmp_bytes(3, 400, 500) > tmp
    for B, H, W in ((0, 8, 8), (-1, 8, 8), (1, 1, 8), (1, 8, 1), (1, 0, 8), (1, 8, -2)):
        assert lib.r3dg_tv_tmp_bytes(B, H, W) == 0
        assert lib.r3dg_tv_forward(B, H, W, p, p, p, 1 << 20, None) == -10001
        assert lib.r3dg_tv_backward(B, H, W, p, p, p, None) == -10001
    for k in range(3):
        ptrs = [p] * 3
        ptrs[k] = None
        assert lib.r3dg_tv_forward(3, 40, 50, ptrs[0], ptrs[1], ptrs[2], tmp, None) == -10001
        assert lib.r3dg_tv_backward(3, 40, 50, *ptrs, None) == -10001
    assert lib.r3dg_tv_forward(3, 40, 50, p, p, p, tmp - 1, None) == -10001
    assert lib.r3dg_tv_forward(65536, 8, 8, p, p, p, 1 << 30, None) == -10002
    assert lib.r3dg_tv_backward(1, 1 << 16, 1 << 15, p, p, p, None) == -10002
    assert lib.r3dg_launch_count() == n0


NAMES = ("ssim", "first_order_edge_aware_loss", "tv_loss")


def _stubs():
    orig = {n: object() for n in NAMES}
    mods = [types.ModuleType(n) for n in ("stub_loss_utils", "stub_render", "stub_neilf")]
    for m in mods:
        for n, v in orig.items():
            setattr(m, n, v)
    return orig, mods


def test_install_by_default_rebinds_only_ssim():
    from relightable3dgaussian_b200 import losses
    orig, mods = _stubs()
    try:
        assert losses.install(*mods) == mods
        for m in mods:
            assert m.ssim is losses.ssim
            assert m.first_order_edge_aware_loss is orig["first_order_edge_aware_loss"] and m.tv_loss is orig["tv_loss"]
    finally:
        losses.uninstall()
    assert all(getattr(m, n) is orig[n] for m in mods for n in NAMES)


def test_install_regularizers_and_uninstall_restores():
    from relightable3dgaussian_b200 import losses
    orig, mods = _stubs()
    bare = types.ModuleType("stub_eval")       # a module that never imported the regularisers
    try:
        losses.install(*mods, regularizers=True)
        losses.install(bare)
        for m in mods:
            assert m.ssim is losses.ssim
            assert m.first_order_edge_aware_loss is losses.first_order_edge_aware_loss
            assert m.tv_loss is losses.tv_loss
        assert bare.ssim is losses.ssim and not hasattr(bare, "tv_loss")
    finally:
        losses.uninstall()
    assert all(getattr(m, n) is orig[n] for m in mods for n in NAMES)
    assert losses.DEFAULT_MODULES == ("utils.loss_utils", "gaussian_renderer.render", "gaussian_renderer.neilf")


def test_rejects_what_the_call_sites_never_pass_without_a_gpu():
    from relightable3dgaussian_b200.losses import first_order_edge_aware_loss, tv_loss
    a = torch.rand(3, 8, 8)
    with pytest.raises(ValueError, match="CUDA"):
        first_order_edge_aware_loss(a, a)
    with pytest.raises(ValueError, match="CUDA"):
        first_order_edge_aware_loss(a.numpy(), a)
    with pytest.raises(ValueError, match="CUDA"):
        tv_loss(a)
