"""Per-pixel (deferred) shading on the GPU: RayTracer.trace_pixels against explicit rays and the bake, and
shading.shade_pixels against `rendering_equation` on the pixels as rows (the row-wise composition of existing kernels),
over image sizes that are not multiples of 16, with and without incidents, transforms, masks and the filtered env."""
import pytest
import torch
import torch.nn.functional as F

import pixel64
from relightable3dgaussian_b200 import synth
from relightable3dgaussian_b200.raytracer import RayTracer, fibonacci_sphere_sampling, inverse_covariance
from relightable3dgaussian_b200.shading import rendering_equation, shade_pixels

pytestmark = pytest.mark.gpu
OUTS = ("pbr", "diffuse_light", "specular")


class SoftplusLight:            # duck-types DirectLightMap (get_env property)
    def __init__(self, env_raw):
        self.env = env_raw

    @property
    def get_env(self):
        return F.softplus(self.env)


class FixedLight:               # duck-types EnvLight (envmap + transform)
    def __init__(self, envmap, transform=None):
        self.envmap, self.transform = envmap, transform


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def scene(P, recipe, seed=5):
    sc = synth.make_scene(P, recipe, seed, 0)
    c = {k: getattr(sc, k).cuda() for k in ("means3D", "scales", "rotations", "opacities", "normals")}
    c["scales"] = c["scales"] * 3.0                                     # more occlusion
    c["inv"] = inverse_covariance(c["scales"], c["rotations"]).contiguous()
    c["opacity"] = c["opacities"][:, 0].contiguous()
    return RayTracer(c["means3D"], c["scales"], c["rotations"]), c


def gbuffer(H, W, V=1, N=16, seed=0):
    """Seeded planar G-buffer of V views (leading V dropped for V = 0): points near the unit shell, blended (not unit)
    normals, materials, incident SH, T in {0} U [0.9, 1], camera centres and rotations."""
    g = torch.Generator().manual_seed(40 + seed)
    lead = (V,) if V else ()
    n = torch.randn(lead + (3, H, W), generator=g)
    pts = F.normalize(torch.randn(lead + (3, H, W), generator=g), dim=-3) * (1 + 0.05 * torch.randn(lead + (1, H, W), generator=g))
    c = dict(normal=n * (0.6 + 0.5 * torch.rand(lead + (1, H, W), generator=g)), points=pts,
             base_color=torch.rand(lead + (3, H, W), generator=g) * 0.8 + 0.05,
             roughness=torch.rand(lead + (1, H, W), generator=g) * 0.9 + 0.08,
             incidents=torch.randn(lead + (48, H, W), generator=g) * 0.3,
             T=torch.where(torch.rand(lead + (N, H, W), generator=g) < 0.3, torch.zeros(lead + (N, H, W)),
                           0.9 + 0.1 * torch.rand(lead + (N, H, W), generator=g)),
             campos=torch.randn(lead + (3,), generator=g) * 3,
             mask=torch.rand(lead + (H, W), generator=g) < 0.7,
             rot=torch.linalg.qr(torch.randn(lead + (3, 3), generator=g, dtype=torch.float64))[0].float(),
             env_raw=torch.randn(1, 16, 32, 3, generator=g))
    c = {k: v.cuda() for k, v in c.items()}
    c["cot"] = {k: torch.randn(lead + (3, H, W), generator=g).cuda() for k in OUTS}
    return c


def rows(t):
    """[C,H,W] -> [HW,C]"""
    return t.reshape(t.shape[0], -1).T.contiguous()


def unit_rows(normal):
    """F.normalize of the [HW,3] rows op by op, as the kernels do."""
    n = rows(normal)
    nn = torch.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2]).clamp_min(1e-12)
    return n / nn[:, None]


def row_shade(c, T, light, incidents, env_filter):
    """rendering_equation on the pixels of one view as rows: (outputs [C,H,W] dict, row leaves)."""
    H, W = c["base_color"].shape[-2:]
    N = T.shape[0]
    dirs, areas = fibonacci_sphere_sampling(unit_rows(c["normal"]), N, random_rotate=False)
    leaves = {"base_color": rows(c["base_color"]).requires_grad_(), "roughness": rows(c["roughness"]).requires_grad_(),
              "incidents": (rows(incidents) if incidents is not None else torch.zeros(H * W, 48, device="cuda"))
              .reshape(-1, 16, 3).requires_grad_()}
    pbr, extra = rendering_equation(leaves["base_color"], leaves["roughness"], rows(c["normal"]),
                                    c["campos"][None] - rows(c["points"]), leaves["incidents"], light, rows(T)[..., None],
                                    dirs, areas, env_filter=env_filter)
    out = {"pbr": pbr, "diffuse_light": extra["diffuse_light"], "specular": extra["specular"]}
    return {k: v.T.reshape(3, H, W) for k, v in out.items()}, leaves


def pixel_shade(c, T, light, incidents, env_filter, mask=None):
    leaves = {"base_color": c["base_color"].clone().requires_grad_(), "roughness": c["roughness"].clone().requires_grad_(),
              "incidents": None if incidents is None else incidents.clone().requires_grad_()}
    out = shade_pixels(leaves["base_color"], leaves["roughness"], c["normal"], c["points"], c["campos"], T, light,
                       incidents=leaves["incidents"], mask=mask, env_filter=env_filter)
    return out, leaves


def loss_of(out, cot):
    return sum((out[k] * cot[k]).sum() for k in OUTS)


# ---- 1. trace = explicit rays, bit for bit ------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W,N,V,recipe,masked", [(1, 1, 8, 0, "shell-v1", False), (13, 29, 32, 0, "cube-v1", True),
                                                   (37, 21, 16, 3, "shell-v1", True), (17, 9, 64, 2, "cube-v1", False)])
def test_trace_equals_explicit_rays(H, W, N, V, recipe, masked):
    rt, s = scene(30_000, recipe)
    c = gbuffer(H, W, V, N)
    mask = c["mask"] if masked else None
    T = rt.trace_pixels(c["points"], c["normal"], N, s["means3D"], s["inv"], s["opacity"], s["normals"], mask=mask)
    assert T.shape == c["points"].shape[:-3] + (N, H, W)
    Tv = T.reshape(-1, N, H, W)
    for v in range(Tv.shape[0]):
        pts = c["points"].reshape(-1, 3, H, W)[v]
        nrm = c["normal"].reshape(-1, 3, H, W)[v]
        dirs, _ = fibonacci_sphere_sampling(unit_rows(nrm), N, random_rotate=False)
        o = rows(pts)[:, None, :].expand(-1, N, -1)
        want = rt.trace_visibility(o, dirs.contiguous(), s["means3D"], s["inv"], s["opacity"], s["normals"])["visibility"][..., 0]
        got = Tv[v].reshape(N, -1).T
        keep = torch.ones(H * W, dtype=torch.bool, device="cuda") if mask is None else mask.reshape(-1, H * W)[v]
        assert bits_equal(got[keep], want[keep])
        assert torch.all(got[~keep] == 0)
    if mask is not None:          # masking changes nothing at the valid pixels
        full = rt.trace_pixels(c["points"], c["normal"], N, s["means3D"], s["inv"], s["opacity"], s["normals"])
        keep = mask.unsqueeze(-3).expand_as(T)
        assert bits_equal(T[keep], full[keep])
    assert ((T == 0) | (T >= 0.9)).all()


def test_pixels_at_gaussians_reproduce_the_bake():
    rt, s = scene(20_000, "shell-v1")
    N = 32
    n = s["normals"]
    nh = n / torch.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2]).clamp_min(1e-12)[:, None]
    fixed = torch.nonzero((nh.view(torch.int32) == n.view(torch.int32)).all(-1))[:, 0][:7 * 11]
    assert fixed.numel() == 77                                         # unit normals whose normalisation keeps their bits
    img = lambda t: t[fixed].T.reshape(3, 7, 11).contiguous()
    T = rt.trace_pixels(img(s["means3D"]), img(n), N, s["means3D"], s["inv"], s["opacity"], n)
    bake = rt.bake_visibility(s["means3D"], s["inv"], s["opacity"], n, N)["visibility"][..., 0]
    assert bits_equal(T.reshape(N, -1).T, bake[fixed])


# ---- 2. shade = the row path -----------------------------------------------------------------------------------------------
SHADE_CASES = [(1, 1, 3, True, False, False), (13, 7, 16, True, True, False), (9, 31, 64, False, False, False),
               (21, 5, 32, True, False, True), (6, 17, 24, False, True, True), (40, 33, 32, True, True, True)]


@pytest.mark.parametrize("H,W,N,with_inc,with_tr,filt", SHADE_CASES)
def test_shade_equals_row_path(H, W, N, with_inc, with_tr, filt):
    c = gbuffer(H, W, 0, N)
    inc = c["incidents"] if with_inc else None
    env_p = c["env_raw"].clone().requires_grad_()
    env_r = c["env_raw"].clone().requires_grad_()
    if with_tr:         # an EnvLight with a transform: gradient to its (activated) envmap
        light_p, light_r = FixedLight(F.softplus(env_p)[0], c["rot"]), FixedLight(F.softplus(env_r)[0], c["rot"])
    else:
        light_p, light_r = SoftplusLight(env_p), SoftplusLight(env_r)
    got, lp = pixel_shade(c, c["T"], light_p, inc, filt)
    want, lr = row_shade(c, c["T"], light_r, inc, filt)
    for k in OUTS:
        assert bits_equal(got[k], want[k]), k
    assert (got["visibility"] - c["T"].mean(0, keepdim=True)).abs().max() < 1e-6
    loss_of(got, c["cot"]).backward()
    loss_of(want, c["cot"]).backward()
    assert rel_l2(lp["base_color"].grad, rows_to_img(lr["base_color"].grad, H, W)) <= 1e-5
    assert rel_l2(lp["roughness"].grad, rows_to_img(lr["roughness"].grad, H, W)) <= 1e-5
    if with_inc:
        assert rel_l2(lp["incidents"].grad, rows_to_img(lr["incidents"].grad.reshape(-1, 48), H, W)) <= 1e-5
    assert env_p.grad.abs().max() > 0 and rel_l2(env_p.grad, env_r.grad) <= 1e-5


def rows_to_img(t, H, W):
    return t.T.reshape(-1, H, W)


@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("H,W,N,filt", [(11, 23, 32, False), (30, 19, 16, True)])
def test_deterministic_env_gradient_bitwise_equal_to_row_path_and_reproducible(H, W, N, filt, det_mode):
    c = gbuffer(H, W, 0, N, seed=2)
    grads = []
    for path in ("pixel", "pixel", "row"):
        env = c["env_raw"].clone().requires_grad_()
        out, leaves = (pixel_shade if path == "pixel" else row_shade)(c, c["T"], SoftplusLight(env), c["incidents"], filt)
        loss_of(out, c["cot"]).backward()
        grads.append((out, leaves, env.grad))
    (o1, l1, e1), (o2, l2, e2), (_, _, e3) = grads
    assert bits_equal(e1, e2) and bits_equal(e1, e3)
    for k in OUTS:
        assert bits_equal(o1[k], o2[k])
    for k in ("base_color", "roughness", "incidents"):
        assert bits_equal(l1[k].grad, l2[k].grad)


# ---- 3. several views --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,H,W,N,filt", [(3, 9, 14, 16, False), (5, 1, 1, 8, True), (2, 23, 17, 32, True)])
def test_views_equal_one_view_calls(V, H, W, N, filt):
    c = gbuffer(H, W, V, N, seed=3)
    tex_v = F.softplus(c["env_raw"])[0].clone().requires_grad_()
    out_v, lv = pixel_shade(c, c["T"], FixedLight(tex_v, c["rot"]), c["incidents"], filt, mask=c["mask"])
    loss_of(out_v, c["cot"]).backward()
    env_sum = torch.zeros_like(tex_v)
    for v in range(V):
        cv = {k: (t[v] if torch.is_tensor(t) else {j: u[v] for j, u in t.items()}) for k, t in c.items() if k != "env_raw"}
        tex = F.softplus(c["env_raw"])[0].clone().requires_grad_()
        out, l1 = pixel_shade(cv, cv["T"], FixedLight(tex, cv["rot"]), cv["incidents"], filt, mask=cv["mask"])
        loss_of(out, cv["cot"]).backward()
        for k in OUTS + ("visibility",):
            assert bits_equal(out_v[k][v], out[k]), (v, k)
        for k in ("base_color", "roughness", "incidents"):
            assert bits_equal(lv[k].grad[v], l1[k].grad), (v, k)
        env_sum += tex.grad
    assert rel_l2(tex_v.grad, env_sum) <= 1e-5


# ---- 4. mask -----------------------------------------------------------------------------------------------------------
def test_masked_pixels_are_zero_and_get_no_gradient():
    c = gbuffer(19, 27, 0, 16, seed=4)
    env = c["env_raw"].clone().requires_grad_()
    out, leaves = pixel_shade(c, c["T"], SoftplusLight(env), c["incidents"], False, mask=c["mask"].to(torch.uint8))
    loss_of(out, c["cot"]).backward()
    off = ~c["mask"]
    for k in OUTS + ("visibility",):
        assert torch.all(out[k][:, off] == 0) and not torch.signbit(out[k][:, off]).any(), k
    for k in ("base_color", "roughness", "incidents"):
        assert torch.all(leaves[k].grad[:, off] == 0), k
    full, _ = pixel_shade(c, c["T"], SoftplusLight(c["env_raw"]), c["incidents"], False)
    for k in OUTS:
        assert bits_equal(out[k][:, c["mask"]], full[k][:, c["mask"]])


# ---- 6. scale ---------------------------------------------------------------------------------------------------------------
def test_1080p_memory_holds_no_per_sample_tensor():
    H, W, N = 1080, 1920, 64
    c = gbuffer(H, W, 0, N, seed=6)
    c["T"] = c["T"].contiguous()
    base = c["base_color"].clone().requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    out = shade_pixels(base, c["roughness"], c["normal"], c["points"], c["campos"], c["T"], SoftplusLight(c["env_raw"]))
    loss_of(out, c["cot"]).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - before
    HW = H * W
    # outputs (10 planes), gradients (4), the loss's products and their cotangents (18), a 64 MB margin
    assert peak <= (10 + 4 + 18) * HW * 4 + (64 << 20), peak / 2**20
    assert peak < HW * N * 3 * 4 / 4                                   # far below one [HW,N,3] tensor


def test_ray_indices_beyond_2_31():
    rt, s = scene(64, "cube-v1")
    H, W, N = 1025, 1025, 2048
    assert H * W * N > 2**31
    g = torch.Generator().manual_seed(11)
    pts = (torch.rand(3, H, W, generator=g) * 2.6 - 1.3).cuda()
    nrm = torch.randn(3, H, W, generator=g).cuda()
    T = rt.trace_pixels(pts, nrm, N, s["means3D"], s["inv"], s["opacity"], s["normals"])
    last = slice(H * W - 1, H * W)
    p_last, n_last = rows(pts)[last], rows(nrm)[last]
    dirs, areas = fibonacci_sphere_sampling(unit_rows(nrm[:, -1:, -1:]), N, random_rotate=False)
    want = rt.trace_visibility(p_last[:, None, :].expand(-1, N, -1), dirs.contiguous(), s["means3D"], s["inv"], s["opacity"],
                               s["normals"])["visibility"][0, :, 0]
    assert bits_equal(T[:, -1, -1], want)
    c = gbuffer(H, W, 0, 1, seed=7)
    tex = F.softplus(c["env_raw"])[0]
    out = shade_pixels(c["base_color"], c["roughness"], nrm, pts, c["campos"], T, FixedLight(tex))
    pbr, _ = rendering_equation(rows(c["base_color"])[last], rows(c["roughness"])[last], n_last, c["campos"][None] - p_last,
                                torch.zeros(1, 16, 3, device="cuda"), FixedLight(tex), want[None, :, None], dirs, areas)
    assert bits_equal(out["pbr"][:, -1, -1], pbr[0])
    del T


# ---- 7. refusals -------------------------------------------------------------------------------------------------------------
def test_refusals():
    rt, s = scene(100, "cube-v1")
    c = gbuffer(5, 6, 0, 8)
    trace = lambda pts, nrm, N: rt.trace_pixels(pts, nrm, N, s["means3D"], s["inv"], s["opacity"], s["normals"])
    with pytest.raises(RuntimeError, match="unsupported"):
        trace(c["points"], c["normal"], 2731)
    with pytest.raises(ValueError, match="views"):
        trace(c["points"].expand(65, 3, 5, 6), c["normal"].expand(65, 3, 5, 6), 8)
    with pytest.raises(ValueError, match="does not match"):
        trace(c["points"], c["normal"][:, :4], 8)
    light = SoftplusLight(c["env_raw"])
    args = [c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], light]
    with pytest.raises(ValueError, match="roughness"):
        shade_pixels(*args[:1], c["base_color"], *args[2:])
    with pytest.raises(ValueError, match="campos"):
        shade_pixels(*args[:4], torch.zeros(2, 3, device="cuda"), *args[5:])
    with pytest.raises(RuntimeError, match="CUDA"):
        shade_pixels(c["base_color"].cpu(), *args[1:])
    big = gbuffer(3, 4, 0, 2731)
    with pytest.raises(RuntimeError, match="unsupported"):
        shade_pixels(big["base_color"], big["roughness"], big["normal"], big["points"], big["campos"], big["T"], light)


# ---- 8. quality: a low-roughness plane under a small bright source -----------------------------------------------------------
def test_quality_of_per_pixel_against_per_gaussian_shading(record_property):
    H, W, N = 48, 64, 256
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1.4, 1.4, W), indexing="ij")
    pts = torch.stack([xs, ys, torch.zeros_like(xs)]).cuda()
    nrm = torch.tensor([0.0, 0.0, 1.0]).view(3, 1, 1).expand(3, H, W).contiguous().cuda()
    base = torch.full((3, H, W), 0.5).cuda()
    rough = torch.full((1, H, W), 0.12).cuda()
    campos = torch.tensor([0.0, -0.6, 1.2]).cuda()
    He = 64
    env = torch.full((He, 2 * He, 3), 0.05)
    env[14:17, 40:44] = 60.0                                            # a small bright source above the horizon
    env = env.cuda()
    T = torch.ones((N, H, W), device="cuda")
    out = shade_pixels(base, rough, nrm, pts, campos, T, FixedLight(env))
    truth = pixel64.shade_pixels(base.cpu(), rough.cpu(), nrm.cpu(), pts.cpu(), campos.cpu(), T.cpu(), env.cpu())["pbr"]
    centre = (slice(None), slice(H // 2, H // 2 + 1), slice(W // 2, W // 2 + 1))
    per_g, _ = rendering_equation(rows(base[centre]), rows(rough[centre]), rows(nrm[centre]), campos[None] - rows(pts[centre]),
                                  torch.zeros(1, 16, 3, device="cuda"), FixedLight(env), torch.ones(1, N, 1, device="cuda"),
                                  *fibonacci_sphere_sampling(rows(nrm[centre]), N, random_rotate=False))
    per_gaussian = per_g[0].view(3, 1, 1).expand(3, H, W).double().cpu()
    err_pixel = rel_l2(out["pbr"].double().cpu(), truth)
    err_gauss = rel_l2(per_gaussian, truth)
    record_property("rel_l2_pixel", err_pixel)
    record_property("rel_l2_per_gaussian", err_gauss)
    print(f"quality: per-pixel rel L2 {err_pixel:.3e}, one Gaussian over the plane {err_gauss:.3e}")
    # fp32 lookup coordinates against fp64 ones at the source's 1200:1 edges: 2.5e-4 measured on an H100
    assert err_pixel <= 1e-3
    assert err_gauss >= 0.1 and err_gauss >= 100 * err_pixel
