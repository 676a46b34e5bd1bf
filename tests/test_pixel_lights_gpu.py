"""GPU per-pixel lights (csrc/lights_trace.cu bvh_pixel_lights_kernel, csrc/pixel_lights.cu): the trace against
trace_lights / trace_shaped_lights rows and the fp64 brute force, the shading against lights.shade / shade_shaped on the
pixels as rows, views, masks, reproducibility, a highlight and a hard shadow that per-Gaussian shading cannot resolve,
and a fit of a point light from a per-pixel image."""
import numpy as np
import pytest
import torch

import lights64 as L64
import pixel_lights64 as PL64
import shaped_lights64 as S64
from helpers import inverse_covariance, npy
from relightable3dgaussian_b200 import lights as lt
from relightable3dgaussian_b200.raytracer import RayTracer
from test_lights_gpu import _case, _leaf_boxes, _lights
from test_shaped_lights_gpu import _mixed

pytestmark = pytest.mark.gpu


def rows(img):
    """[C,H,W] -> [HW,C] (contiguous)."""
    return img.reshape(img.shape[0], -1).T.contiguous()


def gbuffer(V, H, W, R, center, seed=0):
    """Random planar G-buffer images around `center` on the GPU, shadows in [0, 1] and a mask."""
    g = torch.Generator().manual_seed(1300 + seed)
    n = torch.randn(V, 3, H, W, generator=g)
    c = dict(base_color=torch.rand(V, 3, H, W, generator=g) * 0.8 + 0.05,
             roughness=torch.rand(V, 1, H, W, generator=g) * 0.9 + 0.08,
             normal=n * (0.5 + torch.rand(V, 1, H, W, generator=g)),
             points=torch.randn(V, 3, H, W, generator=g) * 0.4 + torch.as_tensor(center).reshape(1, 3, 1, 1),
             campos=torch.randn(V, 3, generator=g) * 0.3 + torch.tensor([0.0, -2.5, 1.7]),
             T=torch.rand(V, R, H, W, generator=g),
             mask=torch.rand(V, H, W, generator=g) < 0.7,
             g_pbr=torch.randn(V, 3, H, W, generator=g), g_diff=torch.randn(V, 3, H, W, generator=g),
             g_spec=torch.randn(V, 3, H, W, generator=g))
    return {k: v.cuda() for k, v in c.items()}


def fields(lights):
    return lt._fields(lights)


def with_grad(lights):
    """A copy of the set whose fields are fresh leaves that require grad."""
    fs = [f.detach().clone().requires_grad_(True) for f in fields(lights)]
    if isinstance(lights, lt.Lights):
        return lt.Lights(lights.kind, *fs)
    return lt.ShapedLights(lights.kind, *fs, M=lights.M, seed=lights.seed)


def point_set(K=6, seed=0):
    g = torch.Generator().manual_seed(seed)
    kind = torch.tensor([j % 2 for j in range(K)], dtype=torch.int32)
    vec = torch.randn(K, 3, generator=g) * 0.6 + torch.tensor([0.0, 0.0, 1.2])
    return lt.Lights(kind, vec.cuda(), (torch.rand(K, 3, generator=g) * 2).cuda())


def shaped_set(M, seed=0):
    c = dict(means3D=torch.tensor([[0.0, 0.0, 1.2], [0.4, -0.3, 1.0], [-0.5, 0.2, 0.9]], device="cuda"))
    return _mixed(c, 3, M, seed)


def row_terms(c, v, lights, T, grads=None):
    """lights.shade / shade_shaped of view v's pixels as rows (viewdirs = campos - points in fp32)."""
    pts = rows(c["points"][v])
    args = (rows(c["base_color"][v]), rows(c["roughness"][v]), rows(c["normal"][v]), c["campos"][v][None] - pts, pts,
            lights, rows(T[v]))
    if grads is not None:
        args = (args[0].requires_grad_(True), args[1].requires_grad_(True)) + args[2:]
    shade = lt.shade if isinstance(lights, lt.Lights) else lt.shade_shaped
    pbr, extra = shade(*args)
    return pbr, extra["diffuse_light"], extra["specular"], args


def rel_l2(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---- 1. trace = the row trace ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("recipe", ["shell-v1", "cube-v1"])
@pytest.mark.parametrize("which", ["points", "M1", "M4", "M8"])
def test_trace_is_the_row_trace(recipe, which):
    """Pixel p holds Gaussian p's mean: T [R,H,W] is trace_lights' / trace_shaped_lights' [P,R] bit for bit."""
    H, W = 48, 64
    P = H * W
    c = _case(recipe, P, seed=21)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"])
    if which == "points":
        lights = _lights(c, 8, 5)
        want = rt.trace_lights(*args, lights)
    else:
        lights = _mixed(c, 3, int(which[1:]), 17)
        want = rt.trace_shaped_lights(*args, lights)
    pts = c["means3D"].T.reshape(3, H, W).contiguous()
    T = rt.trace_pixel_lights(pts, lights, *args)
    R = lt.num_rays(lights)
    assert T.shape == (R, H, W)
    assert (want < 1).any() and (want > 0).any()
    assert torch.equal(T.reshape(R, P).T, want)


# ---- 2. trace vs fp64 -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("recipe", ["shell-v1", "cube-v1"])
@pytest.mark.parametrize("family", ["points", "shaped"])
def test_trace_matches_fp64(recipe, family):
    P, V, H, W = 3000, 2, 12, 10
    c = _case(recipe, P, seed=33)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"])
    lights = _lights(c, 4, 9) if family == "points" else _mixed(c, 3, 2, 19)
    R = lt.num_rays(lights)
    g = gbuffer(V, H, W, R, c["means3D"].mean(0).cpu(), seed=2)
    T = rt.trace_pixel_lights(g["points"], lights, *args, mask=g["mask"])
    assert T.shape == (V, R, H, W)
    keep = g["mask"].cpu().numpy().reshape(V, H * W)
    assert torch.all(T.permute(0, 2, 3, 1)[~g["mask"]] == 0)
    rng = np.random.default_rng(4)
    pixels = [(v, int(p)) for v in range(V) for p in rng.choice(np.flatnonzero(keep[v]), 25, replace=False)]
    T64, fr = PL64.shadows(npy(g["points"]), npy(c["means3D"]), npy(c["inv_cov"]), npy(c["opacity"]), npy(c["normals"]),
                           _leaf_boxes(rt), npy(lights.kind), [npy(f) for f in fields(lights)], getattr(lights, "M", 1),
                           getattr(lights, "seed", 0), pixels)
    Tn = npy(T).reshape(V, R, H * W)
    T64, fr = T64.reshape(V, R, H * W), fr.reshape(V, R, H * W)
    v_idx = np.array([v for v, _ in pixels])[:, None]
    p_idx = np.array([p for _, p in pixels])[:, None]
    r_idx = np.arange(R)[None]
    ok, fragile = L64.shadows_match(Tn[v_idx, r_idx, p_idx], T64[v_idx, r_idx, p_idx], fr[v_idx, r_idx, p_idx])
    print(f"{recipe} {family}: fragile {fragile.mean():.2%}, shadowed {(T64[v_idx, r_idx, p_idx] < 1).mean():.2%}")
    assert (ok | fragile).all()
    assert fragile.mean() <= 0.05


def test_ray_indices_beyond_2_31():
    """V R H W > 2^31 rays (masked pixels decline theirs): the last pixel of the last view equals a one-view call's."""
    c = _case("cube-v1", 64, seed=3)
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"])
    lights = lt.ShapedLights.rect(*(torch.tensor(x, device="cuda").expand(4, 3) for x in
                                    ([0.0, 0.0, 1.5], [0.4, 0.0, 0.0], [0.0, 0.4, 0.0], [1.0, 1.0, 1.0])), M=8, seed=3)
    V, H, W = 2, 2049, 2049
    R = lights.num_rays()
    assert R == 256 and V * R * H * W > 2 ** 31
    g = torch.Generator().manual_seed(5)
    pts = (torch.rand(V, 3, H, W, generator=g) * 2.0 - 1.0).cuda()
    mask = torch.zeros(V, H, W, dtype=torch.bool, device="cuda")
    mask[:, -3:, -3:] = True
    T = rt.trace_pixel_lights(pts, lights, *args, mask=mask)
    last = T[1, :, -1, -1].clone()
    assert torch.all(T[:, :, :-3].eq(0)) and torch.all(T[:, :, :, :-3].eq(0))
    del T
    T1 = rt.trace_pixel_lights(pts[1], lights, *args, mask=mask[1])
    assert torch.equal(last, T1[:, -1, -1])
    p = H * W - 1                                # the oracle's targets hashed with that pixel's index
    tg, _ = S64.ray_targets([3] * 4, *(npy(f) for f in fields(lights)[:3]), 8, 3, p + 1, [p])
    m = np.concatenate([npy(c["means3D"]), npy(pts[1, :, -1, -1])[None]]).astype(np.float32)
    ext = lambda x, y: np.concatenate([x, y]).astype(np.float32)
    T64, fr = L64.shadows(m, ext(npy(c["inv_cov"]), [[1, 0, 0, 1, 0, 1]]), ext(npy(c["opacity"]), [0.0]),
                          ext(npy(c["normals"]), [[0, 0, 1]]), ext(_leaf_boxes(rt), np.tile(m[-1], 2)[None]),
                          np.ones(R, np.int32), tg[p], pairs=[(64, j) for j in range(R)])
    ok, fragile = L64.shadows_match(npy(last), T64[64], fr[64])
    assert (ok | fragile).all()


# ---- 3. shading = the row path ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["points", "M1", "M4"])
@pytest.mark.parametrize("H,W", [(1, 1), (7, 5), (64, 48)])
def test_shading_is_the_row_path(family, H, W):
    lights = with_grad(point_set() if family == "points" else shaped_set(int(family[1:]), seed=H))
    R = lt.num_rays(lights)
    c = gbuffer(1, H, W, R, [0.0, 0.0, 0.0], seed=H * W)
    rl = with_grad(lights)
    pbr, diff, spec, rargs = row_terms(c, 0, rl, c["T"], grads=True)
    b = c["base_color"][0].clone().requires_grad_(True)
    r = c["roughness"][0].clone().requires_grad_(True)
    out = lt.shade_pixels(b, r, c["normal"][0], c["points"][0], c["campos"][0], lights, c["T"][0])
    for k, x in (("pbr", pbr), ("diffuse_light", diff), ("specular", spec)):
        assert out[k].shape == (3, H, W)
        assert torch.equal(rows(out[k]), x), k
    gs = (c["g_pbr"][0], c["g_diff"][0], c["g_spec"][0])
    torch.autograd.backward([pbr, diff, spec], [rows(x) for x in gs])
    torch.autograd.backward([out["pbr"], out["diffuse_light"], out["specular"]], list(gs))
    assert torch.equal(rows(b.grad), rargs[0].grad)
    assert torch.equal(rows(r.grad), rargs[1].grad)
    for fp, fr_ in zip(fields(lights), fields(rl)):
        assert rel_l2(fp.grad, fr_.grad) <= 1e-5 or (fr_.grad.abs().max() == 0 and fp.grad.abs().max() == 0)
    first = [f.grad.clone() for f in fields(lights)] + [b.grad.clone(), r.grad.clone()]
    for f in list(fields(lights)) + [b, r]:
        f.grad = None
    out = lt.shade_pixels(b, r, c["normal"][0], c["points"][0], c["campos"][0], lights, c["T"][0])
    torch.autograd.backward([out["pbr"], out["diffuse_light"], out["specular"]], list(gs))
    for x, y in zip(first, [f.grad for f in fields(lights)] + [b.grad, r.grad]):
        assert torch.equal(x, y)                                   # two runs of the backward are bitwise equal


# ---- 4. views and masks -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["points", "M2"])
def test_views_and_masks(family):
    V, H, W = 3, 19, 23
    lights = with_grad(point_set(seed=1) if family == "points" else shaped_set(2, seed=4))
    R = lt.num_rays(lights)
    c = gbuffer(V, H, W, R, [0.0, 0.0, 0.0], seed=8)
    b = c["base_color"].clone().requires_grad_(True)
    r = c["roughness"].clone().requires_grad_(True)
    out = lt.shade_pixels(b, r, c["normal"], c["points"], c["campos"], lights, c["T"], c["mask"])
    gs = (c["g_pbr"], c["g_diff"], c["g_spec"])
    torch.autograd.backward([out["pbr"], out["diffuse_light"], out["specular"]], list(gs))
    keep = c["mask"][:, None]
    per_view = [torch.zeros_like(f) for f in fields(lights)]
    for v in range(V):
        lv = with_grad(lights)
        bv = c["base_color"][v].clone().requires_grad_(True)
        rv = c["roughness"][v].clone().requires_grad_(True)
        one = lt.shade_pixels(bv, rv, c["normal"][v], c["points"][v], c["campos"][v], lv, c["T"][v], c["mask"][v])
        for k in one:
            assert torch.equal(out[k][v], one[k]), (v, k)
        torch.autograd.backward([one["pbr"], one["diffuse_light"], one["specular"]], [x[v] for x in gs])
        assert torch.equal(b.grad[v], bv.grad) and torch.equal(r.grad[v], rv.grad)
        per_view = [a + f.grad for a, f in zip(per_view, fields(lv))]
    for k in out:
        assert torch.all(out[k].masked_select(~keep) == 0), k
    assert torch.all(b.grad.masked_select(~keep) == 0) and torch.all(r.grad.masked_select(~keep) == 0)
    assert (b.grad != 0).any()
    for f, s in zip(fields(lights), per_view):
        assert rel_l2(f.grad, s) <= 1e-5 or (s.abs().max() == 0 and f.grad.abs().max() == 0)
    if isinstance(lights, lt.Lights):
        # masked pixels add nothing: the light gradients are those of the valid pixels as rows
        rl = with_grad(lights)
        for v in range(V):
            sel = c["mask"][v].reshape(-1)
            pts = rows(c["points"][v])[sel]
            pbr, extra = lt.shade(rows(c["base_color"][v])[sel], rows(c["roughness"][v])[sel], rows(c["normal"][v])[sel],
                                  c["campos"][v][None] - pts, pts, rl, rows(c["T"][v])[sel])
            torch.autograd.backward([pbr, extra["diffuse_light"], extra["specular"]], [rows(x[v])[sel] for x in gs])
        for f, s in zip(fields(lights), fields(rl)):
            assert rel_l2(f.grad, s.grad) <= 1e-5


def test_empty_set_zero_fills():
    c = gbuffer(1, 6, 5, 0, [0.0, 0.0, 0.0])
    empty = lt.Lights(torch.zeros(0, dtype=torch.int32), torch.zeros(0, 3, device="cuda", requires_grad=True),
                      torch.zeros(0, 3, device="cuda"))
    b = c["base_color"][0].clone().requires_grad_(True)
    out = lt.shade_pixels(b, c["roughness"][0], c["normal"][0], c["points"][0], c["campos"][0], empty, c["T"][0])
    assert all(torch.all(x == 0) for x in out.values())
    out["pbr"].sum().backward()
    assert torch.all(b.grad == 0)


# ---- 5. quality -------------------------------------------------------------------------------------------------------------------
def _plane(H, W, extent=1.0, z=0.0):
    ys, xs = torch.meshgrid(torch.linspace(-extent, extent, H), torch.linspace(-extent, extent, W), indexing="ij")
    pts = torch.stack([xs, ys, torch.full_like(xs, z)])
    return pts.cuda(), torch.tensor([0.0, 0.0, 1.0]).reshape(3, 1, 1).expand(3, H, W).contiguous().cuda()


def test_highlight_per_pixel_vs_per_gaussian():
    """A roughness-0.12 plane under a point light: per-pixel pbr is within 2e-4 of fp64 (1.41e-4 measured on an H100
    80GB HBM3 at 700 W); one Gaussian's term spread over the plane is far off (2.85).  The error is the shading step's
    own fp32 GGX, which the pixels share bit for bit with lights.shade: at alpha^2 = 2e-4 its denominator
    NoH^2 (alpha^2 - 1) + 1 cancels to ~alpha^2 at the highlight, amplifying NoH's rounding about 1e4 times."""
    H = W = 128
    pts, nrm = _plane(H, W, 0.5)
    base = torch.full((3, H, W), 0.5, device="cuda")
    rough = torch.full((1, H, W), 0.12, device="cuda")
    campos = torch.tensor([0.3, -0.2, 1.5], device="cuda")
    light = lt.Lights.point(torch.tensor([[-0.1, 0.05, 0.6]], device="cuda"), torch.tensor([[2.0, 2.0, 2.0]], device="cuda"))
    T = torch.ones(1, H, W, device="cuda")
    pix = lt.shade_pixels(base, rough, nrm, pts, campos, light, T)["pbr"]
    ref = PL64.shade_pixels(base[None].cpu(), rough[None].cpu(), nrm[None].cpu(), pts[None].cpu(), campos[None].cpu(),
                            T[None].cpu(), light.kind, (light.vec.cpu(), light.color.cpu()))["pbr"][0]
    err = rel_l2(pix.cpu().double(), ref)
    centre = (slice(None), slice(H // 2, H // 2 + 1), slice(W // 2, W // 2 + 1))
    one = lt.shade_pixels(base[centre], rough[centre], nrm[centre], pts[centre], campos, light, T[centre])["pbr"]
    spread = rel_l2(one.expand(3, H, W).cpu().double(), ref)
    print(f"highlight: per-pixel rel L2 {err:.3e}, one Gaussian spread {spread:.3f}")
    assert err <= 2e-4
    assert spread >= 0.1 and spread >= 100 * err


def _occluder():
    """tests/test_shaped_lights_gpu.py's half-plane: opaque flat Gaussians (spacing and scale 0.01) facing down at
    z = 0.5 over x < 0, and a wide receiver Gaussian (scale 0.05) at the origin facing up."""
    s = 0.01
    xs, ys = np.meshgrid(np.arange(-1.0, 0.0 + 1e-9, s), np.arange(-1.0, 1.0 + 1e-9, s), indexing="ij")
    plane = np.stack([xs.ravel(), ys.ravel(), np.full(xs.size, 0.5)], 1)
    means = np.concatenate([[[0.0, 0.0, 0.0]], plane]).astype(np.float32)
    P = means.shape[0]
    scales = np.tile(np.array([[s, s, s / 10]], np.float32), (P, 1))
    scales[0] = (0.05, 0.05, 0.005)
    rot = np.tile(np.array([[1.0, 0.0, 0.0, 0.0]], np.float32), (P, 1))
    normals = np.tile(np.array([[0.0, 0.0, -1.0]], np.float32), (P, 1))
    normals[0] = (0.0, 0.0, 1.0)
    opacity = np.full(P, 0.99, np.float32)
    opacity[0] = 0.5
    t = lambda x: torch.tensor(x, device="cuda")
    c = dict(means3D=t(means), scales=t(scales), rotations=t(rot), normals=t(normals), opacity=t(opacity))
    c["inv_cov"] = inverse_covariance(c["scales"], c["rotations"])
    return c


def test_hard_shadow_edge_moves_per_pixel():
    c = _occluder()
    rt = RayTracer(c["means3D"], c["scales"], c["rotations"])
    args = (c["means3D"], c["inv_cov"], c["opacity"], c["normals"])
    sun = lt.Lights.directional(torch.tensor([[0.0, 0.0, 1.0]], device="cuda"), torch.ones(1, 3, device="cuda"))
    W = 81                                                       # x from -0.1 to 0.1 in steps of 0.0025
    pts, _ = _plane(3, W, 0.1)
    T = rt.trace_pixel_lights(pts, sun, *args)[0]
    x = pts[0, 0]
    band = 3 * 0.01 + 0.01                                       # 3 sigma of an occluder Gaussian and one spacing
    assert torch.all(T[:, x > band] == 1)
    assert torch.all(T[:, x < -band] < 1e-3)
    edge = T[1, (x.abs() <= band)]
    values = torch.unique(edge[(edge > 1e-3) & (edge < 1)])
    print(f"shadow edge: {values.numel()} distinct T across {int((x.abs() <= band).sum())} pixels of the band")
    assert values.numel() >= 3                                   # the edge moves from pixel to pixel
    Tg = rt.trace_lights(*args, sun)[0]                          # the receiver Gaussian: one value over the whole band
    assert Tg.numel() == 1


# ---- 6. fit --------------------------------------------------------------------------------------------------------------------------
def test_fit_point_light_from_pixels():
    """Adam recovers a point light's position and intensity from a per-pixel image of a glossy plane, re-tracing the
    detached light every step."""
    H = W = 64
    pts, nrm = _plane(H, W, 1.0)
    c = _case("cube-v1", 2000, seed=6)
    scene = {k: v for k, v in c.items()}
    scene["means3D"] = scene["means3D"] * 0.1 + torch.tensor([3.0, 3.0, 0.3], device="cuda")   # a clutter off the plane
    scene["scales"] = scene["scales"] * 0.1
    scene["inv_cov"] = inverse_covariance(scene["scales"], scene["rotations"])
    rt = RayTracer(scene["means3D"], scene["scales"], scene["rotations"])
    args = (scene["means3D"], scene["inv_cov"], scene["opacity"], scene["normals"])
    base = torch.full((3, H, W), 0.5, device="cuda")
    rough = torch.full((1, H, W), 0.3, device="cuda")
    campos = torch.tensor([0.3, -0.2, 2.0], device="cuda")
    true = lt.Lights.point(torch.tensor([[0.2, -0.1, 0.8]], device="cuda"), torch.tensor([[2.0, 1.5, 1.0]], device="cuda"))
    target = lt.shade_pixels(base, rough, nrm, pts, campos, true, rt.trace_pixel_lights(pts, true, *args))["pbr"]
    pos = torch.tensor([[-0.2, 0.2, 1.1]], device="cuda", requires_grad=True)
    col = torch.tensor([[1.0, 1.0, 1.0]], device="cuda", requires_grad=True)
    opt = torch.optim.Adam([pos, col], lr=0.02)
    for step in range(400):
        light = lt.Lights.point(pos, col)
        T = rt.trace_pixel_lights(pts, lt.Lights.point(pos.detach(), col.detach()), *args)
        loss = (lt.shade_pixels(base, rough, nrm, pts, campos, light, T)["pbr"] - target).square().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    dpos = float((pos - true.vec).norm())
    dcol = float(((col - true.color).abs() / true.color).max())
    print(f"fit: position error {dpos:.2e}, intensity error {dcol:.2%}, loss {float(loss):.2e}")
    assert dpos <= 5e-3 and dcol <= 0.01
