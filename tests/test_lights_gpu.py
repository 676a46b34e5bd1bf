"""GPU point and directional lights (csrc/lights_trace.cu, csrc/lights.cu): shadows against their fp64 brute force
(tests/lights64.py) and the trace they share rays with, the shading terms and their gradients against fp64 autograd on
adversarial inputs, against the shading step itself, over several views, reproducibility, and an end-to-end fit."""
import numpy as np
import pytest
import torch

import lights64 as L64
from helpers import inverse_covariance, npy
from relightable3dgaussian_b200 import lights as lt
from relightable3dgaussian_b200 import shading, synth
from relightable3dgaussian_b200.raytracer import RayTracer

pytestmark = pytest.mark.gpu
D = torch.float64


def _case(recipe, P, seed=0):
    sc = synth.make_scene(max(P, 1), recipe, seed, 0)
    normals = -sc.normals if recipe == "shell-v1" else sc.normals
    d = dict(means3D=sc.means3D, scales=sc.scales, rotations=sc.rotations, opacity=sc.opacities[:, 0].contiguous(),
             normals=normals.contiguous(), inv_cov=inverse_covariance(sc.scales, sc.rotations))
    return {k: v[:P].contiguous().cuda() for k, v in d.items()}


def _leaf_boxes(rt):
    P = rt.morton.shape[0]
    boxes = np.empty((P, 6), np.float32)
    boxes[npy(rt.tree[P - 1:, 3]).astype(np.int64)] = npy(rt.aabb[P - 1:])
    return boxes


def _lights(c, K, seed):
    """K lights: alternately directional and point, point lights inside the scene; with K > 1 one point light sits
    exactly at a Gaussian's centre."""
    g = torch.Generator().manual_seed(seed)
    m = c["means3D"].cpu()
    kind = torch.tensor([j % 2 for j in range(K)], dtype=torch.int32)
    vec = torch.randn(K, 3, generator=g)
    inside = m[torch.randint(0, m.shape[0], (K,), generator=g)] + 0.05 * torch.randn(K, 3, generator=g)
    vec = torch.where(kind[:, None] == 1, inside, vec)
    if K > 1:
        vec[1] = m[0]
    color = torch.rand(K, 3, generator=g) * 3
    return lt.Lights(kind, vec.cuda(), color.cuda())


@pytest.mark.parametrize("K", [1, 4, 32])
@pytest.mark.parametrize("P", [1, 2, 500, 3000])
@pytest.mark.parametrize("recipe", ["shell-v1", "cube-v1"])
def test_shadows_match_fp64(recipe, P, K):
    c = _case(recipe, P, seed=P + K)
    lights = _lights(c, K, P * 7 + K)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    T = npy(rt.trace_lights(c["means3D"], c["inv_cov"], c["opacity"], c["normals"], lights))
    assert T.shape == (P, K)
    rays = np.arange(P * K)
    if rays.size > 300:
        rays = np.sort(np.random.default_rng(P * K).choice(rays, 300, replace=False))
    pairs = [(int(r // K), int(r % K)) for r in rays]
    T64, fr = L64.shadows(npy(c["means3D"]), npy(c["inv_cov"]), npy(c["opacity"]), npy(c["normals"]), _leaf_boxes(rt),
                          npy(lights.kind), npy(lights.vec), lone_leaf=P == 1, pairs=pairs)
    g, j = rays // K, rays % K
    ok, fragile = L64.shadows_match(T[g, j], T64[g, j], fr[g, j])
    print(f"{recipe} P={P} K={K}: fragile {fragile.mean():.2%}, shadowed {(T64[g, j] < 1).mean():.2%}, "
          f"differing {(~ok).mean():.2%}")
    assert fragile.mean() <= 0.02
    assert (ok | fragile).all(), (rays[~ok & ~fragile][:5], T[g, j][~ok & ~fragile][:5], T64[g, j][~ok & ~fragile][:5])
    assert np.isfinite(T).all() and (T >= 0).all() and (T <= 1).all()


@pytest.mark.parametrize("recipe", ["shell-v1", "cube-v1"])
def test_directional_shadow_is_the_visibility_trace(recipe):
    """Every Gaussian's ray towards a directional light is the visibility trace's ray (origin mean + 0.05 l,
    RayTracer.trace_visibility) with the same hits in the same order: where that trace keeps T (>= 0.9) the light's T
    is equal bit for bit, where it wrote 0 the light's T is < 0.9.  (The bake itself cannot share one direction over
    Gaussians with distinct normals, and with one shared normal every occluder would be back-facing.)"""
    c = _case(recipe, 20_000, seed=5)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    P = c["means3D"].shape[0]
    for vec in ([0.0, 0.0, 1.0], [0.3, -0.5, 0.7], [-0.8, 0.1, -0.2]):
        v32 = np.asarray(vec, np.float32)
        r2 = np.float32(np.float32(v32[0] * v32[0]) + np.float32(v32[1] * v32[1])) + np.float32(v32[2] * v32[2])
        l = torch.tensor(v32 / np.float32(np.sqrt(np.float32(r2))), device="cuda")   # the kernel's l, op by op
        lights = lt.Lights.directional(torch.tensor([vec], device="cuda"), torch.ones(1, 3, device="cuda"))
        T = rt.trace_lights(c["means3D"], c["inv_cov"], c["opacity"], c["normals"], lights)[:, 0]
        vis = rt.trace_visibility(c["means3D"], l.expand(P, 3).contiguous(), c["means3D"], c["inv_cov"], c["opacity"],
                                  c["normals"])["visibility"][:, 0]
        keep = vis >= 0.9
        assert keep.any() and (~keep).any(), vec
        assert torch.equal(T[keep], vis[keep]), (T[keep] - vis[keep]).abs().max()
        assert bool((T[~keep] < 0.9).all())


def _adversarial(P=512, K=8, seed=0):
    """fp32 inputs covering: a light behind the surface, grazing light, V perpendicular to N (sign 0) and the flipped
    normal, roughness 0 and 1, the GGX nominator clamp, a point light at a Gaussian's centre (R2_MIN) and at 1e4,
    zero colour, and T in {0, 1}."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(P, 3, generator=g)
    rough = torch.rand(P, 1, generator=g)
    rough[::7], rough[1::7] = 0.0, 1.0
    normals = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    normals[2::11] = torch.tensor([0.0, 0.0, 1.0])
    means = torch.randn(P, 3, generator=g) * 0.5
    views = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1)
    views[2::11] = torch.tensor([1.0, 0.0, 0.0])                         # V . N = 0: sign 0
    views[3::11] = -views[3::11]
    kind = torch.tensor([0, 0, 0, 1, 1, 1, 1, 0][:K], dtype=torch.int32)
    vec = torch.tensor([[0.0, 0.0, 1.0], [0.0, 0.0, -1.0], [1.0, 0.0, 1e-4], [0.3, 0.2, 0.4],
                        [1e4, -2e3, 5e3], [0.0, 0.0, 0.0], [0.1, -0.2, 0.3], [-1.0, 2.0, 0.5]][:K])
    color = torch.rand(K, 3, generator=g) * 2
    if K == 8:
        vec[5] = means[5]                                               # a point light at Gaussian 5's centre
        color[6] = 0.0
    T = torch.rand(P, K, generator=g)
    T[::5] = 0.0
    T[1::5] = 1.0
    return base, rough, normals, views, means, kind, vec, color, T


def _run(inputs, V=1, cot=None, seed=1):
    base, rough, normals, views, means, kind, vec, color, T = inputs
    P = base.shape[0]
    g = torch.Generator().manual_seed(seed)
    if views.dim() == 2:
        views = views[None].expand(V, P, 3).contiguous() if V > 1 else views[None]
    leaves = [t.cuda().requires_grad_(True) for t in (base, rough, views, means, vec, color)]
    pbr, extra = lt.shade(leaves[0], leaves[1], normals.cuda(), leaves[2], leaves[3],
                          lt.Lights(kind, leaves[4], leaves[5]), T.cuda())
    outs = (pbr, extra["diffuse_light"], extra["specular"])
    cots = [torch.ones_like(o) if cot == "unit" else torch.randn(o.shape, generator=g).cuda() for o in outs]
    torch.autograd.backward(outs, cots)
    return [o.detach() for o in outs], [t.grad for t in leaves], cots


def _oracle(inputs, views, cots):
    base, rough, normals, _, means, kind, vec, color, T = inputs
    leaves = [t.detach().double().cpu().requires_grad_(True) for t in (base, rough, views, means, vec, color)]
    outs = L64.shade(leaves[0], leaves[1], normals.double(), leaves[2], leaves[3], kind, leaves[4], leaves[5], T.double())
    torch.autograd.backward(outs, [c.double().cpu() for c in cots])
    return [o.detach() for o in outs], [t.grad for t in leaves]


@pytest.mark.parametrize("cot", ["unit", "random"])
def test_shading_and_gradients_match_fp64(cot):
    inputs = _adversarial()
    outs, grads, cots = _run(inputs, cot=cot)
    views = inputs[3][None]
    outs64, grads64 = _oracle(inputs, views, cots)
    for name, a, b in zip(("pbr", "diffuse_light", "specular"), outs, outs64):
        a = a.double().cpu()
        err = (a - b).abs() / (b.abs() + 1e-6)
        assert err.max() < 2e-5, (name, err.max())
    # per-Gaussian rows: each row relative to its own magnitude (rows of a light at the centre carry ~1e20)
    for name, a, b in zip(("base_color", "roughness", "viewdirs", "means3D"), grads[:4], grads64[:4]):
        a, b = a.double().cpu().reshape(b.shape[0] if name != "viewdirs" else b.shape[1], -1), \
            b.reshape(b.shape[0] if name != "viewdirs" else b.shape[1], -1)
        assert torch.isfinite(a).all(), name
        err = (a - b).norm(dim=1) / (b.norm(dim=1) + 1e-6 * b.norm(dim=1).max() + 1e-12)
        assert err.max() < 2e-3, (name, err.max(), int(err.argmax()))
    # the light gradients relative to the sum of the magnitudes of their terms (per-Gaussian autograd rows)
    for name, a, b, leaf in zip(("vec", "color"), grads[4:], grads64[4:], (4, 5)):
        terms = _light_term_magnitudes(inputs, views, cots, leaf)
        err = (a.double().cpu() - b).abs() / (terms + 1e-30)
        assert err.max() < 1e-4, (name, err.max())


def _light_term_magnitudes(inputs, views, cots, leaf):
    """sum over Gaussians of |d(term of Gaussian g)/d(light field)|: the scale the summed light gradient is held to."""
    base, rough, normals, _, means, kind, vec, color, T = inputs
    total = torch.zeros(vec.shape, dtype=D)
    for g in range(base.shape[0]):
        v = vec.double().clone().requires_grad_(leaf == 4)
        c = color.double().clone().requires_grad_(leaf == 5)
        outs = L64.shade(base[g:g + 1].double(), rough[g:g + 1].double(), normals[g:g + 1].double(),
                         views[:, g:g + 1].double(), means[g:g + 1].double(), kind, v, c, T[g:g + 1].double())
        total += torch.autograd.grad(outs, v if leaf == 4 else c, [x.double().cpu()[:, g:g + 1] for x in cots])[0].abs()
    return total


def test_directional_light_is_the_shading_step_with_one_sample():
    P = 4096
    g = torch.Generator().manual_seed(3)
    base, rough = torch.rand(P, 3, generator=g).cuda(), (torch.rand(P, 1, generator=g) * 0.8 + 0.1).cuda()
    normals = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1).cuda()
    views = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=-1).cuda()
    vec = torch.tensor([[0.3, -0.4, 0.8]])
    E = torch.tensor([1.5, 0.7, 2.5])
    T = torch.rand(P, 1, generator=g).cuda()
    lights = lt.Lights.directional(vec.cuda(), E[None].cuda())
    pbr, extra = lt.shade(base, rough, normals, views, torch.randn(P, 3).cuda(), lights, T)
    l = torch.nn.functional.normalize(vec, dim=-1).cuda()

    class Env:
        envmap = E.reshape(1, 1, 3).expand(16, 32, 3).contiguous().cuda()
    ref, rextra = shading.rendering_equation(base, rough, normals, views, torch.zeros(P, 16, 3).cuda(), Env(),
                                             T[:, :, None], l.expand(P, 1, 3).contiguous(), torch.ones(P, 1, 1).cuda())
    for a, b in ((pbr, ref), (extra["diffuse_light"], rextra["diffuse_light"]), (extra["specular"], rextra["specular"])):
        rel = ((a - b).abs() / (b.abs() + 1e-12))[b.abs() > 1e-6]
        assert rel.max() <= 1e-6, rel.max()


@pytest.mark.parametrize("V", [1, 2, 8, 64])
def test_views_equal_one_view_calls(V):
    inputs = _adversarial(P=300, seed=V)
    base, rough, normals, views, means, kind, vec, color, T = inputs
    g = torch.Generator().manual_seed(V)
    vv = torch.nn.functional.normalize(torch.randn(V, 300, 3, generator=g), dim=-1)
    multi = list(inputs)
    multi[3] = vv
    outs, grads, cots = _run(multi, seed=V)
    sums = [torch.zeros_like(x) for x in grads]
    for v in range(V):
        one = list(inputs)
        one[3] = vv[v]
        o1, g1, _ = _run_with(one, [c[v:v + 1] for c in cots])
        for a, b in zip(outs, o1):
            assert torch.equal(a[v], b[0])
        assert torch.equal(grads[2][v], g1[2][0])
        for k in (0, 1, 3, 4, 5):
            sums[k] += g1[k]
    for k in (0, 1, 3):                                   # per-Gaussian rows: the view sums in view order, bit for bit
        assert torch.equal(grads[k], sums[k]), k
    for k in (4, 5):                                      # light gradients: summed in another order
        torch.testing.assert_close(grads[k], sums[k], rtol=1e-4, atol=1e-4 * float(sums[k].abs().max()))


def _run_with(inputs, cots):
    base, rough, normals, views, means, kind, vec, color, T = inputs
    leaves = [t.cuda().requires_grad_(True) for t in (base, rough, views[None], means, vec, color)]
    pbr, extra = lt.shade(leaves[0], leaves[1], normals.cuda(), leaves[2], leaves[3],
                          lt.Lights(kind, leaves[4], leaves[5]), T.cuda())
    outs = (pbr, extra["diffuse_light"], extra["specular"])
    torch.autograd.backward(outs, cots)
    return [o.detach() for o in outs], [t.grad for t in leaves], cots


def test_reproducible_without_the_deterministic_flag():
    assert not torch.are_deterministic_algorithms_enabled()
    inputs = _adversarial(P=100_000, K=8, seed=9)
    a_out, a_grad, _ = _run(inputs, V=4, seed=2)
    b_out, b_grad, _ = _run(inputs, V=4, seed=2)
    assert all(torch.equal(x, y) for x, y in zip(a_out, b_out))
    assert all(torch.equal(x, y) for x, y in zip(a_grad, b_grad))
    c = _case("cube-v1", 20_000, seed=4)
    lights = _lights(c, 8, 4)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"], lights)
    assert torch.equal(rt.trace_lights(*args), rt.trace_lights(*args))


def test_empty_light_set_and_no_gaussians():
    inputs = list(_adversarial(P=64, K=1))
    base, rough, normals, views, means = inputs[:5]
    empty = lt.Lights(torch.zeros(0, dtype=torch.int32), torch.zeros(0, 3).cuda(), torch.zeros(0, 3).cuda())
    leaves = [t.cuda().requires_grad_(True) for t in (base, rough, views, means)]
    pbr, extra = lt.shade(leaves[0], leaves[1], normals.cuda(), leaves[2], leaves[3], empty, torch.zeros(64, 0).cuda())
    assert not pbr.any() and not extra["diffuse_light"].any() and not extra["specular"].any()
    pbr.sum().backward()
    assert all(not t.grad.any() for t in leaves)


def _render(c, pbr, cam, W, H):
    from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    rs = GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, torch.zeros(3, device="cuda"), 1.0,
                                       cam.viewmatrix.cuda(), cam.projmatrix.cuda(), 0, cam.campos.cuda(),
                                       False, False, False, False)
    means2D = torch.zeros_like(c["means3D"], requires_grad=True)
    out = GaussianRasterizer(rs)(means3D=c["means3D"], means2D=means2D, opacities=c["opacity"][:, None],
                                 colors_precomp=pbr, scales=c["scales"], rotations=c["rotations"])
    return out[2]


def test_fit_a_directional_light_through_the_rasterizer():
    """An image rendered with a known sun: Adam on the light's colour and direction, shadows re-traced every step,
    recovers the colour within 2 % and the direction within 2 degrees."""
    c = _case("cube-v1", 20_000, seed=12)
    P = c["means3D"].shape[0]
    W, H = 160, 120
    cam = synth.make_camera(1, W, H)
    base = torch.full((P, 3), 0.6, device="cuda")
    rough = torch.full((P, 1), 0.4, device="cuda")
    views = torch.nn.functional.normalize(cam.campos.cuda()[None] - c["means3D"], dim=-1)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    true = lt.Lights.directional(torch.tensor([[0.4, -0.3, 0.85]], device="cuda"), torch.tensor([[2.0, 1.5, 1.0]], device="cuda"))

    def image(lights):
        T = rt.trace_lights(c["means3D"], c["inv_cov"], c["opacity"], c["normals"],
                            lt.Lights(lights.kind, lights.vec.detach(), lights.color.detach()))
        pbr, _ = lt.shade(base, rough, c["normals"], views, c["means3D"], lights, T)
        return _render(c, pbr + 0.05, cam, W, H)                 # + the shading step's (here constant) env term
    with torch.no_grad():
        target = image(true)
    vec = torch.tensor([[0.55, -0.15, 0.8]], device="cuda", requires_grad=True)
    col = torch.tensor([[1.5, 1.5, 1.5]], device="cuda", requires_grad=True)
    opt = torch.optim.Adam([vec, col], lr=0.02)
    for _ in range(80):
        opt.zero_grad()
        loss = ((image(lt.Lights.directional(vec, col)) - target) ** 2).mean()
        loss.backward()
        opt.step()
    d_true = torch.nn.functional.normalize(true.vec, dim=-1)
    d_fit = torch.nn.functional.normalize(vec.detach(), dim=-1)
    angle = float(torch.rad2deg(torch.arccos((d_true * d_fit).sum().clamp(-1, 1))))
    rel = float(((col.detach() - true.color).abs() / true.color).max())
    print(f"fit: colour rel error {rel:.4f}, direction error {angle:.3f} deg, loss {loss.item():.3e}")
    assert rel < 0.02 and angle < 2.0
