"""rasterize_views refuses what it cannot render before anything is launched (no GPU needed), and the C ABI refuses
several-view calls without their camera table or beyond the view / row limits."""
import ctypes

import pytest
import torch

from relightable3dgaussian_b200 import _lib, rasterizer, synth
from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings, rasterize_views


def _settings(k, W=64, H=48, **kw):
    cam = synth.make_camera(k, W, H)
    s = GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, torch.zeros(3), 1.0,
                                      cam.viewmatrix, cam.projmatrix, 3, cam.campos, False, True, True, False)
    return s._replace(**kw)


def _call(settings, P=10):
    V = len(settings)
    sc = synth.make_scene(P, S=0)
    return rasterize_views(sc.means3D, torch.zeros(V, P, 3), sc.opacities, settings=settings, shs=sc.shs,
                           scales=sc.scales, rotations=sc.rotations)


@pytest.mark.parametrize("field,value", [("image_width", 80), ("image_height", 40), ("sh_degree", 2),
                                         ("scale_modifier", 0.5), ("prefiltered", True),
                                         ("backward_geometry", False), ("computer_pseudo_normal", False)])
def test_settings_that_must_agree(field, value):
    with pytest.raises(ValueError, match=field):
        _call([_settings(0), _settings(1, **{field: value})])


def test_debug_mode_is_refused():
    with pytest.raises(ValueError, match="debug"):
        _call([_settings(0), _settings(1, debug=True)])


def test_installed_gradient_exchange_is_refused():
    rasterizer.set_grad_exchange(object())
    try:
        with pytest.raises(RuntimeError, match="exchange"):
            _call([_settings(0), _settings(1)])
    finally:
        rasterizer.set_grad_exchange(None)


def test_view_and_row_limits():
    with pytest.raises(ValueError, match="at most"):
        _call([_settings(k % 8) for k in range(rasterizer.MAX_VIEWS + 1)])
    with pytest.raises(ValueError, match="means2D"):
        sc = synth.make_scene(10, S=0)
        rasterize_views(sc.means3D, torch.zeros(10, 3), sc.opacities, settings=[_settings(0), _settings(1)],
                        shs=sc.shs, scales=sc.scales, rotations=sc.rotations)


def test_c_abi_refuses_bad_view_arguments():
    lib = _lib.load()
    fake = 0x10000                      # never dereferenced: every call below is refused before anything is enqueued
    cams = (ctypes.c_float * 8)(*([0.3, 0.3, 32.0, 24.0] * 2))
    for V, table, P in ((2, None, 10), (65, cams, 10), (2, cams, 1 << 29)):
        a = _lib.RasterFwdArgs()
        a.P, a.S, a.W, a.H, a.V = P, 0, 64, 48, V
        a.view_cams = ctypes.cast(table, ctypes.c_void_p) if table is not None else None
        a.colors_precomp = a.cov3D_precomp = fake
        assert lib.r3dg_raster_forward(ctypes.byref(a), None) == -10001, (V, P)
    b = _lib.RasterBwdArgs()            # several views with `shs` need the per-view SH factor rows
    b.P, b.S, b.W, b.H, b.V, b.view_cams, b.shs, b.dL_dsh = 10, 0, 64, 48, 2, ctypes.cast(cams, ctypes.c_void_p), fake, fake
    assert lib.r3dg_raster_backward(ctypes.byref(b), None) == -10001


def test_view_sizing_matches_one_view_layout():
    lib = _lib.load()
    for P, S in ((0, 5), (1000, 16)):
        assert lib.r3dg_raster_views_geom_bytes(P, S, 1) == lib.r3dg_raster_geom_bytes(P, S)
        assert lib.r3dg_raster_views_geom_bytes(P, S, 3) > lib.r3dg_raster_geom_bytes(P, S)
    for W, H in ((800, 800), (1920, 1080)):
        assert lib.r3dg_raster_views_img_bytes(W, H, 1) == lib.r3dg_raster_img_bytes(W, H)
        assert lib.r3dg_raster_views_img_n_contrib_offset(W, H, 1) == lib.r3dg_raster_img_n_contrib_offset(W, H)
        assert lib.r3dg_raster_views_img_n_contrib_offset(W, H, 4) >= 4 * W * H * 4
