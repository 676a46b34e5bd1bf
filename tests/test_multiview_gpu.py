"""Multi-view consistency losses on the GPU: against the fp64 oracle on smooth random maps at four sizes, the analytic
plane scene, the chain from rasterize_views(ray_depth=True), bitwise reproducibility in deterministic mode, and
writes confined to the outputs."""
import ctypes

import pytest
import torch

import multiview_oracle as mo
from multiview_check import DEV, TAU, _kernel, _settings, check_against_oracle
from relightable3dgaussian_b200 import _lib, multiview, synth
from relightable3dgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu


def _dev(*ts):
    return [t.float().to(DEV).contiguous() for t in ts]


@pytest.mark.parametrize("WH", [(64, 48), (257, 131), (800, 800), (1080, 1920)])
@pytest.mark.parametrize("pairs", [[(0, 1)], [(0, 1), (1, 0), (0, 2), (1, 1)]], ids=["B1", "B4"])
def test_random_maps_against_fp64_oracle(WH, pairs):
    W, H = WH
    depth, normal, gray, cams = mo.random_scene(W, H, 3, seed=W)
    depth, normal, gray = _dev(depth, normal, gray)
    check_against_oracle(depth, normal, gray, cams, pairs)


def test_plane_scene_on_device():
    """The analytic plane: phi and c are what the CPU oracle finds, so the losses are tiny and agree with it."""
    W, H = 160, 120
    depth, normal, gray, cams = mo.plane_scene(W, H)
    d, n, g = _dev(depth, normal, gray)
    kg, kp, counts = check_against_oracle(d, n, g, cams, [(0, 1), (1, 0)])
    tg, tp = mo.consistency(depth, normal, gray, cams, [(0, 1), (1, 0)])
    assert float(kg.max()) < 1e-3
    assert torch.allclose(kg.double().cpu(), tg, atol=2e-5) and torch.allclose(kp.double().cpu(), tp, atol=2e-4)
    assert int(counts[:, 0].min()) > 0.8 * W * H


def test_end_to_end_from_rasterize_views():
    W, H, S = 160, 120, 5
    sc = synth.make_scene(20000, "shell-v1", 0, S)
    cams = [synth.make_camera(0, W, H), synth.make_camera(0, W, H, elevation_deg=34.0)]
    settings = [R.GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, torch.zeros(3, device=DEV), 1.0,
                                                c.viewmatrix.to(DEV), c.projmatrix.to(DEV), 3, c.campos.to(DEV),
                                                False, True, True, False) for c in cams]
    leaf = lambda t: t.to(DEV).requires_grad_(True)
    means3D, opac, shs, scales, rots, feats = map(leaf, (sc.means3D, sc.opacities, sc.shs, sc.scales, sc.rotations,
                                                         sc.features))
    m2 = torch.zeros(2, means3D.shape[0], 3, device=DEV, requires_grad=True)
    out = R.rasterize_views(means3D, m2, opac, settings=settings, shs=shs, scales=scales, rotations=rots,
                            features=feats, ray_depth=True)
    opacity, depth_img, feature = out[3], out[4], out[5]
    depth = depth_img / opacity.clamp_min(1e-5)
    normal = feature[:, :3]
    gray = mo._smooth(torch.Generator().manual_seed(4), 2, 1, H, W, 6).float().to(DEV).clamp(-1, 1) * 0.2 + 0.5
    pairs = [(0, 1), (1, 0)]
    geo, photo = multiview.consistency_loss(depth, normal, gray, settings, pairs)
    assert torch.isfinite(geo).all() and torch.isfinite(photo).all() and float(geo.detach().sum()) > 0
    depth.retain_grad()
    normal.retain_grad()
    (0.03 * geo.mean() + 0.15 * photo.mean()).backward()
    for name, t in (("means3D", means3D), ("scales", scales), ("rotations", rots), ("opacities", opac)):
        assert t.grad is not None and torch.isfinite(t.grad).all() and float(t.grad.abs().max()) > 0, name
    # the loss and its depth / normal gradients against the oracle on the rendered maps
    mcams = [mo.Cam(c.viewmatrix, c.tanfovx, c.tanfovy, c.cx, c.cy) for c in cams]
    kg, kp, _ = check_against_oracle(depth.detach(), normal.detach().contiguous(), gray, mcams, pairs, border_budget=1e-2)
    assert torch.equal(kg, geo.detach()) and torch.equal(kp, photo.detach())
    assert torch.isfinite(depth.grad).all() and float(normal.grad.abs().max()) > 0


def _det_grads(depth, normal, gray, settings, pairs, det):
    torch.use_deterministic_algorithms(det)
    try:
        cot = (torch.linspace(0.5, 1.5, len(pairs), device=DEV), torch.linspace(1.5, 0.5, len(pairs), device=DEV))
        return _kernel(depth, normal, gray, settings, pairs, cot)[3:]
    finally:
        torch.use_deterministic_algorithms(False)


def test_deterministic_mode_is_bitwise_reproducible():
    W, H = 257, 131
    depth, normal, gray, cams = mo.random_scene(W, H, 3, seed=9)
    d, n, g = _dev(depth, normal, gray)
    settings = _settings(cams, W, H)
    pairs = [(0, 2), (1, 2), (2, 2), (0, 1), (0, 2)]          # a shared neighbour, repeated references and a repeat
    a = _det_grads(d, n, g, settings, pairs, True)
    b = _det_grads(d, n, g, settings, pairs, True)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    c = _det_grads(d, n, g, settings, pairs, False)
    for x, y in zip(a, c):
        assert float((x - y).norm() / y.norm()) < 1e-5


def test_writes_stay_inside_the_outputs_and_zero_depth_gives_zeros():
    W, H, V, B, pad = 96, 64, 2, 1, 4096
    depth, normal, gray, cams = mo.random_scene(W, H, V, seed=2)
    d, n, g = _dev(depth, normal, gray)
    settings = _settings(cams, W, H)
    lib = _lib.load()
    CAN = -12345.5

    def buf(numel, dtype=torch.float32):
        t = torch.full((numel + 2 * pad,), CAN, dtype=torch.float32, device=DEV)
        return t, t[pad:pad + numel]

    for zero in (False, True):
        dd_in = torch.zeros_like(d) if zero else d
        view, cams_h, idx, tau = multiview._prepare(dd_in, n, g, settings, [(0, 1)], TAU)
        geo, geo_v = buf(B)
        photo, photo_v = buf(B)
        cnt, cnt_v = buf(2 * B)
        ddp, ddp_v = buf(V * H * W)
        dnp, dnp_v = buf(V * 3 * H * W)
        cot = torch.ones(B, device=DEV)
        for det in (0, 1):
            a = multiview._args(dd_in, n, g, view, cams_h, idx, tau)
            work = _lib.scratch(lib.r3dg_multiview_work_bytes(B, H, W), DEV)
            a.geo, a.photo, a.counts = geo_v.data_ptr(), photo_v.data_ptr(), cnt_v.data_ptr()
            a.work, a.work_bytes = work.data_ptr(), work.numel()
            _lib.call("r3dg_multiview_forward", DEV, ctypes.byref(a))
            a.dL_dgeo, a.dL_dphoto, a.dL_ddepth, a.dL_dnormal = cot.data_ptr(), cot.data_ptr(), ddp_v.data_ptr(), \
                dnp_v.data_ptr()
            ws = None
            if det:
                ws = _lib.scratch(lib.r3dg_multiview_det_bytes(V, H, W), DEV)
                a.deterministic, a.det_work, a.det_work_bytes = 1, ws.data_ptr(), ws.numel()
            _lib.call("r3dg_multiview_backward", DEV, ctypes.byref(a))
            torch.cuda.synchronize()
            for t, v in ((geo, geo_v), (photo, photo_v), (cnt, cnt_v), (ddp, ddp_v), (dnp, dnp_v)):
                assert bool((t[:pad] == CAN).all()) and bool((t[pad + v.numel():] == CAN).all())
            assert bool((ddp_v != CAN).all()) and bool((dnp_v != CAN).all())
            if zero:
                assert float(geo_v[0]) == 0.0 and float(photo_v[0]) == 0.0
                assert cnt_v.view(torch.int32).tolist() == [0, 0]
                assert bool((ddp_v == 0).all()) and bool((dnp_v == 0).all())
            else:
                assert float(geo_v[0]) > 0 and float(ddp_v.abs().max()) > 0
