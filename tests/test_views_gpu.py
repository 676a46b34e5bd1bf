"""Several views in one call (rasterizer.rasterize_views) against one-view calls of the existing path on the same
inputs: images bit for bit, leaf gradients equal to the fp32 sum of the one-view gradients in view order (bitwise in
deterministic mode), per-view gradients bit for bit."""
import pytest
import torch

from relightable3dgaussian_b200 import _C_raster, synth
from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_views)

pytestmark = pytest.mark.gpu

OUT = ("num_rendered", "n_contrib", "color", "opacity", "depth", "feature", "normal", "surface_xyz", "weights", "radii")
LEAVES = ("means3D", "opacities", "scales", "rotations", "shs", "colors_precomp", "cov3D_precomp", "features")


@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def settings_of(cam, deg=3, bg=None):
    bg = torch.tensor([0.1, 0.4, 0.7]) if bg is None else bg
    return GaussianRasterizationSettings(cam.image_height, cam.image_width, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                         bg.cuda(), 1.0, cam.viewmatrix.cuda(), cam.projmatrix.cuda(), deg,
                                         cam.campos.cuda(), False, True, True, False)


def away_camera(cam):
    """The same camera turned around (every Gaussian of a scene around the origin is behind it: all culled)."""
    view = cam.viewmatrix.double()
    projT = torch.linalg.inv(view) @ cam.projmatrix.double()
    flip = view.clone()
    flip[:, 0] = -flip[:, 0]
    flip[:, 2] = -flip[:, 2]
    return cam._replace(viewmatrix=flip.float().contiguous(), projmatrix=(flip @ projT).float().contiguous())


def make_case(P, W, H, S, V, deg=3, colors=False, cov=False, per_view_features=False, cull=(), seed=0):
    sc = synth.make_scene(P, seed=seed, S=S)
    cams = [synth.make_camera(k, W, H, center_shift=(k % 2 == 1)) for k in range(V)]
    cams = [away_camera(c) if k in cull else c for k, c in enumerate(cams)]
    bgs = [torch.tensor([0.1 * k, 0.5, 1.0 - 0.1 * k]) for k in range(V)]
    settings = [settings_of(c, deg, bg) for c, bg in zip(cams, bgs)]
    g = torch.Generator().manual_seed(seed + 1)
    leaves = dict(means3D=sc.means3D, opacities=sc.opacities)
    if colors:
        leaves["colors_precomp"] = torch.rand(P, 3, generator=g)
    else:
        leaves["shs"] = sc.shs[:, : (deg + 1) ** 2].contiguous() if deg < 3 else sc.shs
    if cov:
        R = _rotation(sc.rotations)
        Sg = R * sc.scales[:, None, :]
        C = Sg @ Sg.transpose(1, 2)
        leaves["cov3D_precomp"] = torch.stack([C[:, 0, 0], C[:, 0, 1], C[:, 0, 2], C[:, 1, 1], C[:, 1, 2], C[:, 2, 2]], 1)
    else:
        leaves["scales"], leaves["rotations"] = sc.scales, sc.rotations
    if S > 0:
        f = sc.features
        leaves["features"] = torch.stack([f + 0.1 * k for k in range(V)]) if per_view_features else f
    leaves = {k: v.cuda().contiguous().requires_grad_(True) for k, v in leaves.items()}
    cot = [dict(color=torch.randn(3, H, W, generator=g), opacity=torch.randn(1, H, W, generator=g),
                depth=torch.randn(1, H, W, generator=g) * 0.1, feature=torch.randn(S, H, W, generator=g))
           for _ in range(V)]
    cot = [{k: t.cuda() for k, t in c.items()} for c in cot]
    return settings, leaves, cot


def _rotation(q):
    q = torch.nn.functional.normalize(q, dim=-1)
    r, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1).view(-1, 3, 3)


def single(settings, leaves, v, m2d):
    kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
    if "features" in kw and kw["features"].dim() == 3:
        kw["features"] = kw["features"][v]
    return dict(zip(OUT, GaussianRasterizer(settings[v])(leaves["means3D"], m2d, leaves["opacities"], **kw)))


def batched(settings, leaves, m2d):
    kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
    return dict(zip(OUT, rasterize_views(leaves["means3D"], m2d, leaves["opacities"], settings=settings, **kw)))


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32) if a.dtype == torch.float32 else a,
                                              b.contiguous().view(torch.int32) if b.dtype == torch.float32 else b)


def check_forward(settings, leaves, det):
    V, P = len(settings), leaves["means3D"].shape[0]
    with torch.no_grad():
        got = batched(settings, leaves, torch.zeros(V, P, 3, device="cuda"))
        for v in range(V):
            ref = single(settings, leaves, v, torch.zeros(P, 3, device="cuda"))
            assert got["num_rendered"][v] == ref["num_rendered"], v
            for k in ("color", "opacity", "depth", "feature", "normal", "surface_xyz", "n_contrib", "radii"):
                assert bits_equal(got[k][v], ref[k]), (k, v)
            if det:
                assert bits_equal(got["weights"][v], ref["weights"]), v
            else:
                torch.testing.assert_close(got["weights"][v], ref["weights"], rtol=1e-3, atol=1e-6)
    return got


def _loss(out, c):
    return sum((out[k] * c[k]).sum() for k in ("color", "opacity", "depth", "feature"))


def grads_single(settings, leaves, cot, scale=1.0):
    """Per-view gradients of the one-view path: ({leaf: [g_0, ..., g_V-1]}, [dL_dmeans2D_v])."""
    V, P = len(settings), leaves["means3D"].shape[0]
    per, m2 = {k: [] for k in leaves}, []
    for v in range(V):
        m2d = torch.zeros(P, 3, device="cuda", requires_grad=True)
        out = single(settings, leaves, v, m2d)
        names = list(leaves)
        gs = torch.autograd.grad(_loss(out, cot[v]) * scale, [leaves[k] for k in names] + [m2d], allow_unused=True)
        for k, g in zip(names, gs[:-1]):
            per[k].append(g)
        m2.append(gs[-1])
    return per, m2


def grads_batched(settings, leaves, cot):
    V, P = len(settings), leaves["means3D"].shape[0]
    m2d = torch.zeros(V, P, 3, device="cuda", requires_grad=True)
    out = batched(settings, leaves, m2d)
    loss = sum(sum((out[k][v] * cot[v][k]).sum() for k in ("color", "opacity", "depth", "feature")) for v in range(V))
    names = list(leaves)
    gs = torch.autograd.grad(loss, [leaves[k] for k in names] + [m2d], allow_unused=True)
    return dict(zip(names, gs[:-1])), gs[-1]


def fold(gs):
    acc = gs[0].clone()
    for g in gs[1:]:
        acc += g
    return acc


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def check_backward(settings, leaves, cot, det):
    per, m2 = grads_single(settings, leaves, cot)
    got, got_m2 = grads_batched(settings, leaves, cot)
    V = len(settings)
    for v in range(V):
        if det:
            assert bits_equal(got_m2[v], m2[v]), ("means2D", v)
        else:
            assert rel_l2(got_m2[v], m2[v]) <= 1e-4, ("means2D", v)
    for k in leaves:
        if leaves[k].dim() == 3 and k == "features":          # per-view input: per-view gradient rows
            for v in range(V):
                ref = per[k][v][v]          # the one-view call read row v of the [V,P,S] leaf
                assert (bits_equal(got[k][v], ref) if det else rel_l2(got[k][v], ref) <= 1e-4), (k, v)
            continue
        ref = fold(per[k])
        if k == "shs" and V > 1:     # rebuilt from the views' rank-1 factors: not bit-identical to the dense sum
            assert rel_l2(got[k], ref) <= 1e-6, (k, rel_l2(got[k], ref))
            assert bool((got[k][ref == 0] == 0).all()), k
            if det:
                again, _ = grads_batched(settings, leaves, cot)
                assert bits_equal(again[k], got[k]), k
        elif det:
            assert bits_equal(got[k], ref), k
        else:
            assert rel_l2(got[k], ref) <= 1e-4, (k, rel_l2(got[k], ref))


@pytest.mark.parametrize("V", [1, 2, 3, 5])
def test_headline_views_forward_and_backward(V, det_mode):
    settings, leaves, cot = make_case(300_000, 800, 800, 5, V)
    check_forward(settings, leaves, det=True)
    check_backward(settings, leaves, cot, det=True)


@pytest.mark.parametrize("V", [2, 3])
def test_default_mode_gradients_within_tolerance(V):
    settings, leaves, cot = make_case(300_000, 800, 800, 5, V)
    check_forward(settings, leaves, det=False)
    check_backward(settings, leaves, cot, det=False)


@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_sh_degrees(deg, det_mode):
    settings, leaves, cot = make_case(100_000, 640, 480, 5, 2, deg=deg)
    check_forward(settings, leaves, det=True)
    check_backward(settings, leaves, cot, det=True)


@pytest.mark.parametrize("per_view", [False, True])
def test_colors_precomp_cov3D_and_features(per_view, det_mode):
    settings, leaves, cot = make_case(100_000, 640, 480, 7, 3, colors=True, cov=True, per_view_features=per_view)
    check_forward(settings, leaves, det=True)
    check_backward(settings, leaves, cot, det=True)


def test_per_view_colors_precomp(det_mode):
    settings, leaves, cot = make_case(100_000, 640, 480, 5, 3, colors=True)
    leaves["colors_precomp"] = torch.stack([leaves["colors_precomp"].detach() * (0.5 + 0.2 * k) for k in range(3)]
                                           ).contiguous().requires_grad_(True)
    V, P = 3, 100_000
    with torch.no_grad():
        got = batched(settings, leaves, torch.zeros(V, P, 3, device="cuda"))
        for v in range(V):
            one = dict(leaves, colors_precomp=leaves["colors_precomp"][v])
            ref = single(settings, one, v, torch.zeros(P, 3, device="cuda"))
            assert bits_equal(got["color"][v], ref["color"]), v
    gb, _ = grads_batched(settings, leaves, cot)
    for v in range(V):
        one = dict(leaves, colors_precomp=leaves["colors_precomp"][v].detach().clone().requires_grad_(True))
        out = single(settings, one, v, torch.zeros(P, 3, device="cuda"))
        (g,) = torch.autograd.grad(_loss(out, cot[v]), [one["colors_precomp"]])
        assert bits_equal(gb["colors_precomp"][v], g), v


def test_culled_view_next_to_normal_views(det_mode):
    settings, leaves, cot = make_case(100_000, 640, 480, 5, 3, cull=(1,))
    got = check_forward(settings, leaves, det=True)
    assert got["num_rendered"][1] == 0 and got["num_rendered"][0] > 0 and got["num_rendered"][2] > 0
    check_backward(settings, leaves, cot, det=True)


def test_no_gaussians():
    settings, leaves, cot = make_case(0, 320, 240, 5, 3)
    got = check_forward(settings, leaves, det=False)
    assert got["num_rendered"] == [0, 0, 0]


def test_first_call_overflows_its_binning_buffer(det_mode):
    settings, leaves, _ = make_case(100_000, 640, 480, 5, 3)
    rs = settings[0]
    with torch.no_grad():
        args = (torch.stack([s.bg for s in settings]), leaves["means3D"], leaves["features"], None, leaves["opacities"],
                leaves["scales"], leaves["rotations"], 1.0, None, torch.stack([s.viewmatrix for s in settings]),
                torch.stack([s.projmatrix for s in settings]), [(s.tanfovx, s.tanfovy, s.cx, s.cy) for s in settings],
                rs.image_height, rs.image_width, leaves["shs"], 3, torch.stack([s.campos for s in settings]), False, True)
        out = _C_raster.rasterize_views(*args, _min_capacity=4096)      # far below the instance count: re-run
        assert out[11].numel() > _C_raster._lib.load().r3dg_raster_binning_bytes(4096)
        for v in range(3):
            ref = single(settings, leaves, v, torch.zeros(100_000, 3, device="cuda"))
            assert out[0][v] == ref["num_rendered"]
            assert bits_equal(out[2][v], ref["color"]) and bits_equal(out[1][v], ref["n_contrib"]), v


def test_large_grids_forward():
    # 1.5M Gaussians, 1600x1200, S = 16, 8 views (60 000 tiles) and 1920x1080 with a partial last tile row per view
    settings, leaves, _ = make_case(1_500_000, 1600, 1200, 16, 8)
    check_forward(settings, leaves, det=False)
    del settings, leaves
    settings, leaves, _ = make_case(300_000, 1920, 1080, 5, 8)
    check_forward(settings, leaves, det=False)


@pytest.mark.parametrize("det", [False, True])
def test_mean_of_view_losses_step(det):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        settings, leaves, _ = make_case(200_000, 640, 480, 5, 3, seed=7)
        g = torch.Generator().manual_seed(11)
        targets = [torch.rand(3, 480, 640, generator=g).cuda() for _ in range(3)]
        V, P = 3, 200_000
        names = list(leaves)
        m2d = torch.zeros(V, P, 3, device="cuda", requires_grad=True)
        out = batched(settings, leaves, m2d)
        loss = sum((out["color"][v] - targets[v]).abs().mean() + 0.1 * out["depth"][v].mean() for v in range(V)) / V
        got = torch.autograd.grad(loss, [leaves[k] for k in names])
        per = {k: [] for k in names}
        for v in range(V):
            o = single(settings, leaves, v, torch.zeros(P, 3, device="cuda", requires_grad=True))
            lv = ((o["color"] - targets[v]).abs().mean() + 0.1 * o["depth"].mean()) / V
            for k, gk in zip(names, torch.autograd.grad(lv, [leaves[k] for k in names])):
                per[k].append(gk)
        for k, gk in zip(names, got):
            ref = fold(per[k])
            if k == "shs":
                assert rel_l2(gk, ref) <= (1e-6 if det else 1e-4), k
            elif det:
                assert bits_equal(gk, ref), k
            else:
                assert rel_l2(gk, ref) <= 1e-4, (k, rel_l2(gk, ref))
    finally:
        torch.use_deterministic_algorithms(prev)
