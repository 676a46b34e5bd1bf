"""GPU spot and rect lights (csrc/lights_trace.cu, csrc/lights.cu): shadows against their fp64 brute force
(tests/shaped_lights64.py) and against trace_lights' point lights at the same points, a penumbra, the shading terms and
every gradient against fp64 autograd, views, reproducibility, empty cases and an end-to-end fit of a rect light."""
import numpy as np
import pytest
import torch

import lights64 as L64
import shaped_lights64 as S64
from helpers import inverse_covariance, npy
from relightable3dgaussian_b200 import lights as lt
from relightable3dgaussian_b200 import synth
from relightable3dgaussian_b200.raytracer import RayTracer
from test_lights_gpu import _case, _leaf_boxes, _render

pytestmark = pytest.mark.gpu
D = torch.float64


def _mixed(c, K, M, seed):
    """K lights alternately spot and rect inside the scene, rects of random size and orientation."""
    g = torch.Generator().manual_seed(seed)
    m = c["means3D"].cpu()
    pos = m[torch.randint(0, m.shape[0], (K,), generator=g)] + 0.05 * torch.randn(K, 3, generator=g)
    a = torch.randn(K, 3, generator=g) * 0.1
    b = torch.randn(K, 3, generator=g) * 0.1
    kind = torch.tensor([2 + j % 2 for j in range(K)], dtype=torch.int32)
    cone = torch.stack([torch.full((K,), 0.9), torch.full((K,), 0.5)], -1)
    color = torch.rand(K, 3, generator=g) * 3
    return lt.ShapedLights(kind, pos.cuda(), a.cuda(), b.cuda(), color.cuda(), cone.cuda(), M=M, seed=seed)


@pytest.mark.parametrize("P, K, M", [(2, 1, 4), (3000, 1, 4), (3000, 8, 4), (3000, 3, 8), (100_000, 8, 4)])
@pytest.mark.parametrize("recipe", ["shell-v1", "cube-v1"])
def test_shadows_match_fp64(recipe, P, K, M):
    c = _case(recipe, P, seed=P + K)
    lights = _mixed(c, K, M, P * 7 + K)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    T = npy(rt.trace_shaped_lights(c["means3D"], c["inv_cov"], c["opacity"], c["normals"], lights))
    R = lights.num_rays()
    assert T.shape == (P, R)
    rays = np.arange(P * R)
    if rays.size > 200:
        rays = np.sort(np.random.default_rng(P * K).choice(rays, 200, replace=False))
    pairs = [(int(r // R), int(r % R)) for r in rays]
    T64, fr = S64.shadows(npy(c["means3D"]), npy(c["inv_cov"]), npy(c["opacity"]), npy(c["normals"]), _leaf_boxes(rt),
                          npy(lights.kind), npy(lights.pos), npy(lights.a), npy(lights.b), M, lights.seed, pairs,
                          lone_leaf=P == 1)
    g, j = rays // R, rays % R
    ok, fragile = L64.shadows_match(T[g, j], T64[g, j], fr[g, j])
    print(f"{recipe} P={P} K={K} M={M}: fragile {fragile.mean():.2%}, shadowed {(T64[g, j] < 1).mean():.2%}, "
          f"differing {(~ok).mean():.2%}")
    assert (ok | fragile).all(), (rays[~ok & ~fragile][:5], T[g, j][~ok & ~fragile][:5], T64[g, j][~ok & ~fragile][:5])
    # at 100k Gaussians a shadow ray passes within rounding of some decision far more often (tens of occluders each)
    assert fragile.mean() <= (0.03 if P <= 3000 else 0.3)
    assert np.isfinite(T).all() and (T >= 0).all() and (T <= 1).all()


@pytest.mark.parametrize("recipe", ["shell-v1", "cube-v1"])
def test_spot_shadow_is_the_point_light_shadow(recipe):
    c = _case(recipe, 20_000, seed=2)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    spots = _mixed(c, 1, 1, 3)
    args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"])
    T = rt.trace_shaped_lights(*args, spots)
    Tp = rt.trace_lights(*args, lt.Lights.point(spots.pos, torch.ones_like(spots.pos)))
    assert (T < 1).any()
    assert torch.equal(T, Tp)


@pytest.mark.parametrize("M", [2, 4, 8])
def test_rect_sample_shadows_are_point_light_shadows(M):
    """For chosen Gaussians, point lights at that Gaussian's M^2 sample points (the oracle's fp32 points) give, through
    trace_lights, its row of the rect's shadows bit for bit: the trace's points are the oracle's, hash included."""
    c = _case("cube-v1", 20_000, seed=4)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"])
    rect = lt.ShapedLights.rect(c["means3D"][10:11] + 0.1, torch.tensor([[0.2, 0.0, 0.05]], device="cuda"),
                                torch.tensor([[0.0, 0.15, 0.0]], device="cuda"), torch.ones(1, 3, device="cuda"), M=M, seed=77)
    T = rt.trace_shaped_lights(*args, rect)
    P = c["means3D"].shape[0]
    rows = [0, 1, 5000, 12345, P - 1]
    tg, _ = S64.ray_targets([3], npy(rect.pos), npy(rect.a), npy(rect.b), M, rect.seed, P, rows)
    shadowed = 0
    for g in rows:
        for lo in range(0, M * M, 32):
            pts = torch.tensor(tg[g, lo:lo + 32], device="cuda")
            Tp = rt.trace_lights(*args, lt.Lights.point(pts, torch.ones_like(pts)))
            assert torch.equal(T[g, lo:lo + 32], Tp[g]), (g, lo)
            shadowed += int((Tp[g] < 1).sum())
    print(f"M={M}: {shadowed} of {len(rows) * M * M} rays shadowed")


def _adversarial(P=256, M=2, seed=0):
    """Mixed lights over adversarial materials: roughness 0 and 1, V perpendicular to N, a light behind, a spot at a
    Gaussian's centre, a spot with cos_inner = cos_outer, a degenerate rect, T in {0, 1}."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(P, 3, generator=g)
    rough = torch.rand(P, 1, generator=g)
    rough[::7], rough[1::7] = 0.0, 1.0
    normals = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    normals[2::11] = torch.tensor([0.0, 0.0, 1.0])
    means = torch.randn(P, 3, generator=g) * 0.5
    views = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    views[2::11] = torch.tensor([1.0, 0.0, 0.0])
    kind = torch.tensor([2, 3, 2, 3, 3, 2], dtype=torch.int32)
    pos = torch.tensor([[0.0, 0.0, 1.5], [0.2, -0.3, 1.2], [0.0, 0.0, 0.0], [-1.0, 0.5, 0.2], [0.5, 0.5, 2.0],
                        [1.0, -1.0, 1.0]])
    pos[2] = means[5]
    a = torch.tensor([[0.1, 0.0, -1.0], [0.3, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.2, 0.1], [0.2, 0.0, 0.0],
                      [-1.0, 1.0, -1.0]])
    b = torch.tensor([[0.0, 0.0, 0.0], [0.0, 0.2, 0.05], [0.0, 0.0, 0.0], [0.25, 0.0, 0.0], [0.4, 0.0, 0.0],
                      [0.0, 0.0, 0.0]])                                  # light 4: u parallel to v, degenerate
    cone = torch.tensor([[0.9, 0.6], [0.0, 0.0], [0.5, 0.2], [0.0, 0.0], [0.0, 0.0], [0.8, 0.8]])
    color = torch.rand(6, 3, generator=g) * 2
    R = 3 + 3 * M * M
    T = torch.rand(P, R, generator=g)
    T[::5] = 0.0
    T[1::5] = 1.0
    return base, rough, normals, views, means, kind, pos, a, b, color, cone, T, M


def _run(inputs, views, cots=None, cot="random", seed=1):
    base, rough, normals, _, means, kind, pos, a, b, color, cone, T, M = inputs
    g = torch.Generator().manual_seed(seed)
    leaves = [t.cuda().requires_grad_(True) for t in (base, rough, views, means, pos, a, b, color, cone)]
    lights = lt.ShapedLights(kind, *leaves[4:], M=M, seed=seed + 10)
    pbr, extra = lt.shade_shaped(leaves[0], leaves[1], normals.cuda(), leaves[2], leaves[3], lights, T.cuda())
    outs = (pbr, extra["diffuse_light"], extra["specular"])
    if cots is None:
        cots = [torch.ones_like(o) if cot == "unit" else torch.randn(o.shape, generator=g).cuda() * 1e-3 for o in outs]
    torch.autograd.backward(outs, cots)
    return [o.detach() for o in outs], [t.grad for t in leaves], cots, lights


def _oracle(inputs, views, cots, seed, rows=None):
    base, rough, normals, _, means, kind, pos, a, b, color, cone, T, M = inputs
    rows = slice(None) if rows is None else rows
    P = base.shape[0]
    _, st = S64.ray_targets(kind.tolist(), pos, a, b, M, seed, P)
    leaves = [t.detach().double().cpu().requires_grad_(True)
              for t in (base[rows], rough[rows], views[:, rows], means[rows], pos, a, b, color, cone)]
    outs = S64.shade(leaves[0], leaves[1], normals[rows].double(), leaves[2], leaves[3], kind.tolist(), *leaves[4:],
                     T[rows].double(), M, st[rows])
    torch.autograd.backward(outs, [c.double().cpu()[:, rows] for c in cots])
    return [o.detach() for o in outs], [t.grad for t in leaves]


@pytest.mark.parametrize("cot", ["unit", "random"])
def test_shading_and_gradients_match_fp64(cot):
    inputs = _adversarial()
    views = inputs[3][None]
    outs, grads, cots, lights = _run(inputs, views, cot=cot)
    outs64, grads64 = _oracle(inputs, views, cots, lights.seed)
    for name, x, y in zip(("pbr", "diffuse_light", "specular"), outs, outs64):
        err = (x.double().cpu() - y).abs() / (y.abs() + 1e-6)
        assert err.max() < 2e-4, (name, err.max())           # GGX near roughness 0 amplifies fp32 rounding of l
    for name, x, y in zip(("base_color", "roughness", "viewdirs", "means3D"), grads[:4], grads64[:4]):
        x = x.double().cpu().reshape(-1, 3 if name != "roughness" else 1)
        y = y.reshape(x.shape)
        assert torch.isfinite(x).all(), name
        err = (x - y).norm(dim=1) / (y.norm(dim=1) + 1e-6 * y.norm(dim=1).max() + 1e-12)
        assert err.max() < 2e-3, (name, err.max(), int(err.argmax()))
    # the light gradients, relative to the sum over Gaussians of the magnitudes of their terms
    P = inputs[0].shape[0]
    mags = [torch.zeros_like(x) for x in grads64[4:]]
    for g in range(P):
        _, gg = _oracle(inputs, views, cots, lights.seed, rows=slice(g, g + 1))
        for k in range(5):
            mags[k] += gg[4 + k].abs()
    for name, x, y, mag in zip(("pos", "a", "b", "color", "cone"), grads[4:], grads64[4:], mags):
        assert torch.isfinite(x).all(), name
        err = (x.double().cpu() - y).abs() / (mag + 1e-30)
        assert err.max() < 1e-4, (name, err.max())
    assert grads[6][[0, 2, 5]].abs().max() == 0 and grads[8][[1, 3, 4]].abs().max() == 0   # unused fields


@pytest.mark.parametrize("V", [1, 8])
def test_views_equal_one_view_calls(V):
    inputs = _adversarial(P=300, seed=V)
    g = torch.Generator().manual_seed(V)
    vv = torch.nn.functional.normalize(torch.randn(V, 300, 3, generator=g), dim=-1)
    outs, grads, cots, _ = _run(inputs, vv, seed=V)
    sums = [torch.zeros_like(x) for x in grads]
    for v in range(V):
        o1, g1, _, _ = _run(inputs, vv[v:v + 1], cots=[c[v:v + 1] for c in cots], seed=V)
        for x, y in zip(outs, o1):
            assert torch.equal(x[v], y[0])
        assert torch.equal(grads[2][v], g1[2][0])
        for k in (0, 1, 3, 4, 5, 6, 7, 8):
            sums[k] += g1[k]
    for k in (0, 1, 3):
        assert torch.equal(grads[k], sums[k]), k
    for k in (4, 5, 6, 7, 8):
        torch.testing.assert_close(grads[k], sums[k], rtol=1e-4, atol=1e-4 * float(sums[k].abs().max()) + 1e-30)


@pytest.mark.parametrize("deterministic", [False, True])
def test_reproducible(deterministic):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        inputs = _adversarial(P=100_000, M=4, seed=9)
        vv = torch.nn.functional.normalize(torch.randn(4, 100_000, 3), dim=-1)
        a_out, a_grad, cots, _ = _run(inputs, vv, seed=2)
        b_out, b_grad, _, _ = _run(inputs, vv, cots=cots, seed=2)
        assert all(torch.equal(x, y) for x, y in zip(a_out, b_out))
        assert all(torch.equal(x, y) for x, y in zip(a_grad, b_grad))
        c = _case("cube-v1", 20_000, seed=4)
        lights = _mixed(c, 8, 4, 4)
        rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
        args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"], lights)
        assert torch.equal(rt.trace_shaped_lights(*args), rt.trace_shaped_lights(*args))
    finally:
        torch.use_deterministic_algorithms(prev)


def test_empty_light_set_and_no_gaussians():
    inputs = _adversarial(P=64)
    base, rough, normals, views, means = inputs[:5]
    z = torch.zeros(0, 3).cuda()
    empty = lt.ShapedLights(torch.zeros(0, dtype=torch.int32), z, z, z, z, torch.zeros(0, 2).cuda())
    leaves = [t.cuda().requires_grad_(True) for t in (base, rough, views, means)]
    pbr, extra = lt.shade_shaped(leaves[0], leaves[1], normals.cuda(), leaves[2], leaves[3], empty, torch.zeros(64, 0).cuda())
    assert not pbr.any() and not extra["diffuse_light"].any() and not extra["specular"].any()
    pbr.sum().backward()
    assert all(not t.grad.any() for t in leaves)
    # P = 0 with lights: nothing shaded, zero light gradients
    _, _, _, _, _, kind, pos, a, b, color, cone, _, M = inputs
    lv = [t.cuda().requires_grad_(True) for t in (pos, a, b, color, cone)]
    lights = lt.ShapedLights(kind, *lv, M=M)
    e3 = torch.zeros(0, 3).cuda()
    pbr, _ = lt.shade_shaped(e3, torch.zeros(0, 1).cuda(), e3, e3, e3, lights, torch.zeros(0, lights.num_rays()).cuda())
    assert pbr.shape == (0, 3)
    (pbr.sum() + sum(t.sum() * 0 for t in lv)).backward()
    assert all(not t.grad.any() for t in lv)


def _plane_scene():
    """A receiver at the origin facing up and an opaque plane of small flat Gaussians facing down at z = 0.5, covering
    x < 0."""
    s = 0.01
    xs, ys = np.meshgrid(np.arange(-1.0, 0.0 + 1e-9, s), np.arange(-1.0, 1.0 + 1e-9, s), indexing="ij")
    plane = np.stack([xs.ravel(), ys.ravel(), np.full(xs.size, 0.5)], 1)
    means = np.concatenate([[[0.0, 0.0, 0.0]], plane]).astype(np.float32)
    P = means.shape[0]
    scales = np.tile(np.array([[s, s, s / 10]], np.float32), (P, 1))
    scales[0] = 0.001
    rot = np.tile(np.array([[1.0, 0.0, 0.0, 0.0]], np.float32), (P, 1))
    normals = np.tile(np.array([[0.0, 0.0, -1.0]], np.float32), (P, 1))
    normals[0] = (0.0, 0.0, 1.0)
    opacity = np.full(P, 0.99, np.float32)
    opacity[0] = 0.5
    t = lambda x: torch.tensor(x, device="cuda")
    c = dict(means3D=t(means), scales=t(scales), rotations=t(rot), normals=t(normals), opacity=t(opacity))
    c["inv_cov"] = inverse_covariance(c["scales"], c["rotations"])
    return c


def test_penumbra():
    """Half of a rect hidden by the plane: the receiver's rays are about half blocked.  A point light just past the
    plane's edge, or just behind it, gives a hard 1 or 0."""
    c = _plane_scene()
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"])
    rect = lt.ShapedLights.rect(torch.tensor([[0.0, 0.0, 1.0]], device="cuda"), torch.tensor([[0.0, 0.3, 0.0]], device="cuda"),
                                torch.tensor([[0.3, 0.0, 0.0]], device="cuda"), torch.ones(1, 3, device="cuda"), M=8, seed=1)
    T = rt.trace_shaped_lights(*args, rect)[0]
    print(f"receiver T mean {float(T.mean()):.3f}, fractional {int(((T > 1e-3) & (T < 1)).sum())} of 64")
    assert 0.4 <= float(T.mean()) <= 0.6
    pts = torch.tensor([[0.1, 0.0, 1.0], [-0.1, 0.0, 1.0]], device="cuda")
    Tp = rt.trace_lights(*args, lt.Lights.point(pts, torch.ones_like(pts)))[0]
    assert float(Tp[0]) == 1.0 and float(Tp[1]) < 1e-3


def test_fit_a_rect_light_through_the_rasterizer():
    """An image rendered under a known softbox: Adam on its centre and radiance, shadows re-traced every step,
    recovers the centre within 2 % of the scene size and the radiance within 3 %."""
    c = _case("cube-v1", 20_000, seed=12)
    P = c["means3D"].shape[0]
    W, H = 160, 120
    cam = synth.make_camera(1, W, H)
    base = torch.full((P, 3), 0.6, device="cuda")
    rough = torch.full((P, 1), 0.4, device="cuda")
    views = torch.nn.functional.normalize(cam.campos.cuda()[None] - c["means3D"], dim=-1)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    lo, hi = c["means3D"].min(0).values, c["means3D"].max(0).values
    size = float((hi - lo).norm())
    mid = (lo + hi) / 2
    u = torch.tensor([[0.0, 0.15, 0.0]], device="cuda") * size
    v = torch.tensor([[0.15, 0.0, 0.0]], device="cuda") * size                  # u x v = -z: emits downwards
    true_pos = (mid + torch.tensor([0.1, -0.05, 0.6], device="cuda") * size)[None]
    true_rad = torch.tensor([[2.0, 1.5, 1.0]], device="cuda")

    def image(pos, rad):
        lights = lt.ShapedLights.rect(pos, u, v, rad, M=4, seed=3)
        T = rt.trace_shaped_lights(c["means3D"], c["inv_cov"], c["opacity"], c["normals"],
                                   lt.ShapedLights.rect(pos.detach(), u, v, rad.detach(), M=4, seed=3))
        pbr, _ = lt.shade_shaped(base, rough, c["normals"], views, c["means3D"], lights, T)
        return _render(c, pbr + 0.05, cam, W, H)
    with torch.no_grad():
        target = image(true_pos, true_rad)
    pos = (true_pos + torch.tensor([[-0.06, 0.05, 0.08]], device="cuda") * size).clone().requires_grad_(True)
    rad = torch.tensor([[1.5, 1.5, 1.5]], device="cuda", requires_grad=True)
    opt = torch.optim.Adam([{"params": [pos], "lr": 0.005 * size}, {"params": [rad], "lr": 0.02}])
    for _ in range(150):
        opt.zero_grad()
        loss = ((image(pos, rad) - target) ** 2).mean()
        loss.backward()
        opt.step()
    dpos = float((pos.detach() - true_pos).norm()) / size
    drad = float(((rad.detach() - true_rad).abs() / true_rad).max())
    print(f"fit: centre error {dpos:.4f} of the scene size, radiance rel error {drad:.4f}, loss {loss.item():.3e}")
    assert dpos < 0.02 and drad < 0.03
