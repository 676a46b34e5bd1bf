"""Appearance-only rasterizer backward without a GPU: the C layer's refusals of mixed geometry outputs before any
launch, and the host layer's refusal of camera gradients in that mode."""
import ctypes

import pytest
import torch

from relightable3dgaussian_b200 import _C_raster, _lib

FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued
GEOMETRY_OUTPUTS = ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dscales", "dL_drotations")


def _bwd_args(lib, P=100, S=5, W=64, H=48):
    a = _lib.RasterBwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(W, H)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    a.dL_dfeatures = FAKE
    return a


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5])
def test_mixed_null_geometry_outputs_are_refused(n):
    lib = _lib.load()
    for first in range(len(GEOMETRY_OUTPUTS)):
        a = _bwd_args(lib)
        for k in range(n):
            setattr(a, GEOMETRY_OUTPUTS[(first + k) % len(GEOMETRY_OUTPUTS)], FAKE)
        assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001, (n, first)


def test_camera_gradient_without_geometry_outputs_is_refused():
    lib = _lib.load()
    a = _bwd_args(lib)
    a.dL_dviewmatrix = a.dL_dprojmatrix = a.dL_dcampos = FAKE
    a.cam_work, a.cam_work_bytes = FAKE, lib.r3dg_raster_cam_grad_bytes(100, 1)
    assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001


def test_appearance_backward_with_nothing_requested_is_refused():
    lib = _lib.load()
    a = _bwd_args(lib)
    a.dL_dfeatures = None
    assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001
    a.P = 0                           # no Gaussians: nothing to do, refused for none of the combinations
    assert lib.r3dg_raster_backward(ctypes.byref(a), None) == 0


def test_host_refuses_camera_gradients_in_the_appearance_backward():
    P, H, W = 4, 8, 8
    z = lambda *s: torch.zeros(*s)
    with pytest.raises(ValueError, match="appearance-only"):
        _C_raster.rasterize_gaussians_backward(
            z(3), z(P, 3), z(P, 5), None, torch.Tensor([]), z(P, 3), z(P, 4), 1.0, torch.Tensor([]), torch.eye(4),
            torch.eye(4), 1.0, 1.0, z(3, H, W), z(1, H, W), z(1, H, W), z(5, H, W), z(P, 16, 3), 3, z(3), None, 0, None,
            None, True, False, cam_grads=True, geometry=False)
