"""Camera gradients without a GPU: the C layer's refusals before any launch, the workspace sizing, and the refusal of
camera gradients under an installed gradient exchange."""
import ctypes

import pytest
import torch

from relightable3dgaussian_b200 import _lib
from relightable3dgaussian_b200 import rasterizer as R

FAKE = 0x10000      # never dereferenced: every call below is refused before anything is enqueued


def _bwd_args(lib, P=100, S=5, W=64, H=48):
    a = _lib.RasterBwdArgs()
    a.P, a.S, a.W, a.H = P, S, W, H
    a.geom, a.geom_bytes = FAKE, lib.r3dg_raster_geom_bytes(P, S)
    a.img, a.img_bytes = FAKE, lib.r3dg_raster_img_bytes(W, H)
    a.binning, a.binning_bytes = FAKE, lib.r3dg_raster_binning_bytes(10_000)
    return a


def test_cam_grad_bytes_exact():
    """35 floats per view and per CTA of 128 Gaussians, rounded up to 256 bytes; P = 0 and V < 1 are sized as 1."""
    lib = _lib.load()
    want = {(0, 1): 256, (1, 1): 256, (128, 1): 256, (129, 1): 512, (-5, 0): 256, (1000, 1): 1280,
            (1000, 3): 3584, (10**6, 1): 1093888, (10**6, 8): 8750592, (1_500_000, 1): 1640704,
            (1_500_000, 64): 105002240}
    got = {k: lib.r3dg_raster_cam_grad_bytes(*k) for k in want}
    assert got == want
    for P, V in want:
        blocks = (max(P, 1) + 127) // 128
        assert got[(P, V)] == -(-max(V, 1) * 35 * blocks * 4 // 256) * 256


@pytest.mark.parametrize("given", [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (0, 1, 1), (1, 0, 1)])
def test_partial_camera_outputs_are_refused(given):
    lib = _lib.load()
    for P in (100, 0):
        a = _bwd_args(lib, P=P)
        a.cam_work, a.cam_work_bytes = FAKE, lib.r3dg_raster_cam_grad_bytes(P, 1)
        a.dL_dviewmatrix, a.dL_dprojmatrix, a.dL_dcampos = (FAKE if g else None for g in given)
        assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001, (P, given)


def test_too_small_camera_workspace_is_refused():
    lib = _lib.load()
    for P, V in ((100, 1), (0, 1), (1000, 3)):
        a = _bwd_args(lib, P=P)
        if V > 1:
            cams = (ctypes.c_float * (4 * V))(*([1.0, 1.0, 32.0, 24.0] * V))
            a.V, a.view_cams = V, ctypes.cast(cams, ctypes.c_void_p)
            a.geom_bytes = lib.r3dg_raster_views_geom_bytes(P, 5, V)
            a.img_bytes = lib.r3dg_raster_views_img_bytes(64, 48, V)
        a.dL_dviewmatrix = a.dL_dprojmatrix = a.dL_dcampos = FAKE
        a.cam_work, a.cam_work_bytes = FAKE, lib.r3dg_raster_cam_grad_bytes(P, V) - 1
        assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001, (P, V)
        a.cam_work, a.cam_work_bytes = None, lib.r3dg_raster_cam_grad_bytes(P, V)
        assert lib.r3dg_raster_backward(ctypes.byref(a), None) == -10001, (P, V)


def test_pack_features_viewmatrix_gradient_refusals():
    """dL_dviewmatrix needs the depth channels and a workspace of r3dg_raster_cam_grad_bytes(P, 1) bytes."""
    lib = _lib.load()
    P, S = 1000, 4
    arr = (_lib.PackSrc * 1)()
    arr[0].ptr, arr[0].width = None, 2
    need = lib.r3dg_raster_cam_grad_bytes(P, 1)
    call = lambda m, v, work, nbytes: lib.r3dg_pack_features_backward(P, S, m, v, FAKE, 1, arr, None, FAKE, work, nbytes,
                                                                      None)
    assert call(FAKE, FAKE, FAKE, need - 1) == -10001          # too small
    assert call(FAKE, FAKE, None, need) == -10001              # no workspace
    arr[0].width = 4
    assert call(None, None, FAKE, need) == -10001              # no depth channels to differentiate


def test_camera_grad_refused_under_grad_exchange(monkeypatch):
    """An installed gradient exchange renders one view per rank; a camera tensor that requires grad is refused before
    the forward runs."""
    called = []
    monkeypatch.setattr(R._C, "rasterize_gaussians", lambda *a, **k: called.append(1))
    P, H, W = 7, 4, 5
    means3D, means2D, opac, shs = torch.randn(P, 3), torch.zeros(P, 3), torch.rand(P, 1), torch.randn(P, 16, 3)
    scales, rots = torch.rand(P, 3), torch.randn(P, 4)
    for which in ("viewmatrix", "projmatrix", "campos"):
        cam = dict(viewmatrix=torch.eye(4), projmatrix=torch.eye(4), campos=torch.zeros(3))
        cam[which].requires_grad_(True)
        rs = R.GaussianRasterizationSettings(H, W, 1.0, 1.0, 0.0, 0.0, torch.zeros(3), 1.0, cam["viewmatrix"],
                                             cam["projmatrix"], 3, cam["campos"], False, True, True, False)
        R.set_grad_exchange(object(), torch.zeros(1, 3))
        try:
            with pytest.raises(RuntimeError, match="gradient exchange"):
                R.GaussianRasterizer(rs)(means3D=means3D, means2D=means2D, opacities=opac, shs=shs, scales=scales,
                                         rotations=rots)
        finally:
            R.set_grad_exchange(None)
    assert not called
