"""Multi-view consistency losses without a GPU: the fp64 oracle's identities (a view against itself, an analytic
tilted plane, finite differences) and the refusals of multiview.consistency_loss and of the C ABI, which all happen
before anything touches a device."""
import ctypes

import pytest
import torch

import multiview_oracle as mo
from relightable3dgaussian_b200 import _lib, multiview
from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings


def _interior(e, W, H, margin=6):
    q = e["q"]
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    xs, ys = xs.reshape(-1), ys.reshape(-1)
    return (e["geo"] & (q[:, 0] > margin) & (q[:, 0] < W - 1 - margin) & (q[:, 1] > margin) & (q[:, 1] < H - 1 - margin)
            & (xs >= 3) & (xs < W - 3) & (ys >= 3) & (ys < H - 3))


def test_a_view_against_itself_has_zero_loss():
    """Pair (v, v) with an exactly orthonormal fp64 camera: phi = 0, and ncc = 1 up to its 1e-8 regulariser, i.e.
    c = 1 - var(a) / sqrt(var(a)^2 + 1e-8) at every pixel."""
    W, H = 64, 48
    depth, normal, gray, cams = mo.plane_scene(W, H)
    cams = [mo.Cam(mo.look_at((3.0, 1.0, 2.5)), c.tanfovx, c.tanfovy, c.cx, c.cy) for c in cams]
    depth = torch.stack([mo.plane_depth(c, W, H, (0.15, -0.1, 1.0))[0] for c in cams])[:, None]
    geo, photo, (e,) = mo.consistency(depth, normal, gray, cams, [(0, 0)], info=True)
    inner = torch.zeros(H, W, dtype=torch.bool)
    inner[1:-1, 1:-1] = True                      # on the border q may round to just outside the image
    assert bool(e["geo"][inner.reshape(-1)].all())
    assert float(e["phi"][e["geo"]].max()) < 1e-9
    assert float(geo[0]) < 1e-9
    a = torch.nn.functional.pad(gray[0, 0], (3, 3, 3, 3)).unfold(0, 7, 1).unfold(1, 7, 1).reshape(H * W, 49)
    va = a.var(-1, unbiased=False)
    want = 1 - va / torch.sqrt(va * va + mo.NCC_EPS)
    sel = e["geo"]
    assert float((e["c"][sel] - want[sel]).abs().max()) < 1e-9
    assert float(photo[0]) < 1e-3


@pytest.mark.parametrize("WH", [(96, 72), (160, 120)])
def test_plane_scene_is_consistent(WH):
    """Two cameras on an analytic tilted plane with a smooth texture: phi < 1e-2 px and c < 1e-2 at interior pixels
    (not tighter: bilinear interpolation of z and of the image is not exact on a plane)."""
    W, H = WH
    depth, normal, gray, cams = mo.plane_scene(W, H)
    geo, photo, infos = mo.consistency(depth, normal, gray, cams, [(0, 1), (1, 0)], info=True)
    for e in infos:
        inter = _interior(e, W, H)
        assert int(inter.sum()) > 0.5 * W * H
        assert float(e["phi"][inter].max()) < 1e-2
        assert float(e["c"][inter].max()) < 1e-2
    assert float(geo.max()) < 1e-3          # the photometric mean also holds border patches that leave the image


def test_perturbed_depth_raises_geo_and_gradient_matches_finite_differences():
    W, H = 20, 16
    depth, normal, gray, cams = mo.random_scene(W, H, 2, seed=3)
    pairs = [(0, 1), (1, 0), (0, 1)]           # (v, v) would put its border pixels on the image-bound decision
    # from consistent maps (the analytic plane, phi ~ 0), a perturbation of view 0's depth raises both pairs' geo
    pd, pn, pg, pc = mo.plane_scene(W, H)
    base, _ = mo.consistency(pd, pn, pg, pc, pairs)
    g = torch.Generator().manual_seed(1)
    bumped = pd.clone()
    bumped[0] *= 1 + 0.002 * torch.randn(1, H, W, generator=g, dtype=torch.float64)
    geo, _ = mo.consistency(bumped, pn, pg, pc, pairs)
    assert float(geo[0]) > 3 * float(base[0]) and float(geo[1]) > 3 * float(base[1])

    # the counts of the unperturbed maps are held fixed, and no pixel lies within 1e-4 of a decision boundary, so the
    # loss is smooth in a neighbourhood of these maps
    _, _, infos = mo.consistency(depth, normal, gray, cams, pairs, info=True)
    for e in infos:
        gb, pb = mo.borderline(e, 1.0, W, H, delta=1e-4)
        assert not bool(gb.any()) and not bool(pb.any())
    counts = [(int(e["geo"].sum()), int(e["photo"].sum())) for e in infos]
    weights = [e["w"] for e in infos]       # w = exp(-phi) has no gradient: held at the base maps' values
    wsum = torch.tensor([0.7, -0.4, 1.3, 0.9, 0.5, -1.1], dtype=torch.float64)

    def f(d, n):
        geo, photo = mo.consistency(d, n, gray, cams, pairs, counts=counts, weights=weights)
        return (torch.cat([geo, photo]) * wsum).sum()

    d0, n0 = depth.clone().requires_grad_(), normal.clone().requires_grad_()
    gd, gn = torch.autograd.grad(f(d0, n0), [d0, n0])
    assert float(gd.abs().max()) > 0 and float(gn.abs().max()) > 0
    for k in range(3):                     # central differences along random directions
        vd = torch.randn(depth.shape, generator=g, dtype=torch.float64) * depth
        vn = torch.randn(normal.shape, generator=g, dtype=torch.float64)
        h = 1e-7
        with torch.no_grad():
            fd = (f(depth + h * vd, normal + h * vn) - f(depth - h * vd, normal - h * vn)) / (2 * h)
        an = (gd * vd).sum() + (gn * vn).sum()
        assert float((fd - an).abs()) <= 1e-5 * float(an.abs()) + 1e-9, (k, float(fd), float(an))


def _settings(W, H, V=2, tanfovx=0.5):
    return [GaussianRasterizationSettings(H, W, tanfovx, tanfovx * H / W, W / 2, H / 2, torch.zeros(3), 1.0,
                                          torch.eye(4), torch.eye(4), 0, torch.zeros(3), False, True, True, False)
            for _ in range(V)]


def test_refusals_happen_on_the_host():
    W, H = 16, 12
    d, n, g = torch.ones(2, 1, H, W), torch.ones(2, 3, H, W), torch.ones(2, 1, H, W)
    s = _settings(W, H)
    cl = multiview.consistency_loss
    with pytest.raises(TypeError, match="float32"):
        cl(d.double(), n, g, s, [(0, 1)])
    with pytest.raises(ValueError, match=r"\[V,3,H,W\]"):
        cl(d, n[:, :2], g, s, [(0, 1)])
    with pytest.raises(ValueError, match="disagrees"):
        cl(d, n, g[:, :, :-1], s, [(0, 1)])
    with pytest.raises(ValueError, match="settings for"):
        cl(d, n, g, s[:1], [(0, 1)])
    with pytest.raises(ValueError, match="the maps are"):
        cl(d, n, g, _settings(W + 1, H), [(0, 1)])
    with pytest.raises(ValueError, match="outside"):
        cl(d, n, g, s, [(0, 2)])
    with pytest.raises(ValueError, match="outside"):
        cl(d, n, g, s, [(-1, 0)])
    with pytest.raises(ValueError, match="pairs per call"):
        cl(d, n, g, s, [])
    with pytest.raises(ValueError, match="pairs per call"):
        cl(d, n, g, s, [(0, 1)] * 65)
    with pytest.raises(TypeError, match="two ints"):
        cl(d, n, g, s, [(0, 1.0)])
    with pytest.raises(ValueError, match="pixel_noise_threshold"):
        cl(d, n, g, s, [(0, 1)], pixel_noise_threshold=float("nan"))
    with pytest.raises(ValueError, match="CUDA"):          # every host check passed: only the device is missing
        cl(d, n, g, s, [(0, 1)])


FAKE = 0x10000          # never dereferenced: every call below is refused before anything is enqueued


def test_c_abi_refuses_before_any_launch():
    lib = _lib.load()
    assert lib.r3dg_multiview_work_bytes(0, 8, 8) == 0 and lib.r3dg_multiview_work_bytes(65, 8, 8) == 0
    assert lib.r3dg_multiview_work_bytes(2, 48, 64) == 768            # 2 pairs x 12 CTAs x 4 doubles
    assert lib.r3dg_multiview_work_bytes(4, 1080, 1920) == 4 * 68 * 120 * 32
    assert lib.r3dg_multiview_det_bytes(2, 48, 64) >= 2 * 4 * 48 * 64 * 24
    cams = (ctypes.c_float * 16)(*([0.5, 0.4, 32.0, 24.0] * 4))
    pairs = (ctypes.c_int * 4)(0, 1, 1, 0)

    def args(**kw):
        a = _lib.MultiviewArgs()
        a.V, a.H, a.W, a.B = 2, 48, 64, 2
        a.depth = a.normal = a.gray = a.viewmatrix = FAKE
        a.pair_cams, a.pairs = ctypes.addressof(cams), ctypes.addressof(pairs)
        a.pixel_noise_threshold = 1.0
        a.geo = a.photo = a.counts = a.work = FAKE
        a.work_bytes = lib.r3dg_multiview_work_bytes(2, 48, 64)
        a.dL_dgeo = a.dL_dphoto = a.dL_ddepth = a.dL_dnormal = FAKE
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    fwd, bwd = lib.r3dg_multiview_forward, lib.r3dg_multiview_backward
    for kw in ({"B": 0}, {"B": 65}, {"V": 0}, {"W": 0}, {"depth": None}, {"pairs": None}, {"pair_cams": None},
               {"work_bytes": 255}, {"geo": None}, {"pixel_noise_threshold": -1.0}, {"V": 1}):
        assert fwd(ctypes.byref(args(**kw)), None) == -10001, kw
    for kw in ({"dL_ddepth": None}, {"counts": None}, {"deterministic": 1}, {"V": 1},
               {"deterministic": 1, "det_work": FAKE, "det_work_bytes": 1024}):
        assert bwd(ctypes.byref(args(**kw)), None) == -10001, kw
    cams[1] = 0.0                                                         # tan_fovy <= 0
    assert fwd(ctypes.byref(args()), None) == -10001
    cams[1] = float("inf")
    assert fwd(ctypes.byref(args()), None) == -10001
    cams[1] = 0.4
    pairs[3] = 2                                                          # neighbour index outside [0, V)
    assert fwd(ctypes.byref(args()), None) == -10001
    assert fwd(None, None) == -10001 and bwd(None, None) == -10001
