"""Importance-sampled environment lighting on the GPU: the env table and the sampler against the fp64 oracle
(importance64.py), the importance bake against trace_visibility, and the shading step under the sampler against the
quadrature truth of the plane-under-a-source scene, values and gradients."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import importance64 as I
from relightable3dgaussian_b200 import synth
from relightable3dgaussian_b200.raytracer import RayTracer, fibonacci_sphere_sampling, inverse_covariance
from relightable3dgaussian_b200.shading import (EnvSampler, importance_sample, rendering_equation, rendering_equation_views,
                                                shade_pixels)

pytestmark = pytest.mark.gpu


class FixedLight:               # duck-types EnvLight (envmap + transform)
    def __init__(self, envmap, transform=None):
        self.envmap, self.transform = envmap, transform


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def random_env(He, We, seed):
    g = np.random.default_rng(seed)
    env = g.gamma(0.5, 1.0, (He, We, 3))
    env[He // 3, We // 4] = 500.0
    return env


def rotation(seed):
    return np.linalg.qr(np.random.default_rng(seed).standard_normal((3, 3)))[0]


def rows(P, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.randn(P, 3, generator=g)
    v = n + 1.5 * torch.randn(P, 3, generator=g)
    r = torch.rand(P, 1, generator=g) * 0.9 + 0.08
    return n.cuda(), v.cuda(), r.cuda()


# ---- table --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("He,We", [(2, 2), (2, 3), (17, 40), (64, 128), (300, 601)])
def test_table_matches_the_oracle(He, We):
    env = random_env(He, We, He + We)
    s = EnvSampler(FixedLight(torch.tensor(env, dtype=torch.float32).cuda()))
    tab = s.table.cpu().numpy()
    assert tab[:2].view(np.int32).tolist() == [He, We]
    got = I.from_gpu_table(tab, He, We)
    want = I.build_table(env.astype(np.float32).astype(np.float64))
    for k in ("row_cdf", "vers", "covers", "col_cdf"):
        assert np.abs(got[k] - want[k]).max() <= 1e-6, k
    # the pdfs from the GPU's own CDFs (one rounding of the CDFs can move a small cell's pdf by more than 1e-6)
    pdf = np.diff(got["row_cdf"])[:, None] * np.diff(got["col_cdf"], axis=1) / I.cell_solid_angle(He, We)[:, None]
    assert np.all(np.abs(got["pdf"] - pdf) <= 1e-6 * np.abs(pdf) + 1e-30)
    s2 = EnvSampler(FixedLight(torch.tensor(env, dtype=torch.float32).cuda()))
    assert bits_equal(s.table, s2.table)                                       # bitwise reproducible


def test_zero_env_table_is_uniform():
    s = EnvSampler(FixedLight(torch.zeros(16, 33, 3, device="cuda")))
    got = I.from_gpu_table(s.table.cpu().numpy(), 16, 33)
    assert np.abs(got["pdf"] * 4 * math.pi - 1).max() <= 1e-4


# ---- sampler ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mix,with_tr", [((0.5, 0.25, 0.25), False), ((0.5, 0.25, 0.25), True), ((0.0, 0.0, 1.0), False),
                                         ((0.7, 0.0, 0.3), True), ((0.2, 0.6, 0.2), True)])
def test_directions_and_areas_match_the_oracle(mix, with_tr):
    He, We, P, N = 32, 64, 700, 32
    env = random_env(He, We, 7)
    T = rotation(3) if with_tr else None
    light = FixedLight(torch.tensor(env, dtype=torch.float32).cuda(), None if T is None else torch.tensor(T, dtype=torch.float32).cuda())
    s = EnvSampler(light, mix=mix, seed=11)
    n, v, r = rows(P, 1)
    dirs, areas = importance_sample(n, s, N, v, r)
    tab = I.from_gpu_table(s.table.cpu().numpy(), He, We)
    Tt = None if T is None else light.transform.double().cpu().numpy()
    ne, ng, _ = s.counts(N)
    d64, a64, edge = I.sample(tab, Tt, n.double().cpu().numpy(), N, ne, ng, 11, viewdirs=v.double().cpu().numpy(),
                              roughness=r.double().cpu().numpy()[:, 0])
    nz = F.normalize(n, dim=-1)[:, 2].cpu().numpy()
    _, Ns, _ = I.ggx_frame(I.normalize(n.double().cpu().numpy()), v.double().cpu().numpy(), r.double().cpu().numpy()[:, 0])
    # rotate_from_z divides by 1 + z of its axis (the normal, or the flipped normal of the GGX samples), which amplifies
    # fp32 rounding by ~1 / (1 + z): the tolerance scales with it, and axes within 0.1 of -z are left out.  Samples
    # within 1e-5 rad of an env cell edge may take the neighbouring cell's pdf.
    z = np.minimum(nz, Ns[:, 2]) if ng > 0 else nz
    keep = (z > -0.9)[:, None] & (edge > 1e-5)
    tol = (2e-6 * np.maximum(1.0, 0.5 / (1.0 + np.maximum(z, -0.9))))[:, None]
    d = dirs.double().cpu().numpy()
    assert np.all((np.abs(d - d64).max(-1) <= tol)[keep])
    a = areas[..., 0].double().cpu().numpy()
    rel = (np.abs(a - a64) / (np.abs(a64) + 1e-30))[keep]
    print(f"area rel err: median {np.median(rel):.2e}, 99.9% {np.quantile(rel, 0.999):.2e}, max {rel.max():.2e}")
    if ng == 0:
        assert np.quantile(rel, 0.999) <= 1e-5 and rel.max() <= 1e-4
    else:
        # The GGX pdf of a narrow lobe is limited by fp32 h itself: h = normalize(V + l) is rounded to ~1e-7 rad, and at
        # roughness 0.08 the lobe is ~6e-3 rad wide, so D(h) moves by ~1e-4 relative (more for the narrowest rows).  D's
        # denominator is formed without cancellation; measured on an H100: median 5e-8 - 2e-7, 99.9 % 2.5e-4 - 7.6e-4.
        assert np.median(rel) <= 1e-6 and np.quantile(rel, 0.999) <= 2e-3
    assert keep.mean() > 0.85


def test_same_seed_same_bits_other_seed_other_samples():
    env = torch.tensor(random_env(16, 32, 2), dtype=torch.float32).cuda()
    n, v, r = rows(100, 2)
    a = importance_sample(n, EnvSampler(FixedLight(env), seed=5), 16, v, r)
    b = importance_sample(n, EnvSampler(FixedLight(env), seed=5), 16, v, r)
    c = importance_sample(n, EnvSampler(FixedLight(env), seed=6), 16, v, r)
    assert bits_equal(a[0], b[0]) and bits_equal(a[1], b[1])
    assert not torch.equal(a[0], c[0])


# ---- bake ---------------------------------------------------------------------------------------------------------------
def test_bake_importance_equals_trace_visibility():
    sc = synth.make_scene(3000, "shell-v1", 5, 0)
    c = {k: getattr(sc, k).cuda() for k in ("means3D", "scales", "rotations", "opacities", "normals")}
    inv = inverse_covariance(c["scales"] * 3.0, c["rotations"]).contiguous()
    rt = RayTracer(c["means3D"], c["scales"] * 3.0, c["rotations"])
    op = c["opacities"][:, 0].contiguous()
    s = EnvSampler(FixedLight(torch.tensor(random_env(32, 64, 4), dtype=torch.float32).cuda()))
    P = c["means3D"].shape[0]
    v = torch.randn(P, 3, device="cuda")
    r = torch.rand(P, 1, device="cuda")
    out = rt.bake_importance(c["means3D"], inv, op, c["normals"], s, 32, v, r)
    dirs, areas = importance_sample(c["normals"], s, 32, v, r)
    assert bits_equal(out["incident_dirs"], dirs) and bits_equal(out["incident_areas"], areas)
    ref = rt.trace_visibility(c["means3D"][:, None].expand(-1, 32, -1), dirs, c["means3D"], inv, op, c["normals"])
    assert bits_equal(out["visibility"], ref["visibility"])
    assert 0.05 < float((out["visibility"] == 0).float().mean()) < 0.95        # the scene occludes some rays


# ---- quality and gradients on the plane ----------------------------------------------------------------------------------
PIXELS = [(24, 32), (24, 10), (24, 50), (10, 32), (40, 32), (5, 5)]


def plane_rows(rough):
    env = torch.tensor(I.plane_env(), dtype=torch.float32).cuda()
    pts = np.stack([I.plane_pixel(y=y, x=x)[0] for y, x in PIXELS])
    cam = I.plane_pixel()[2]
    M = len(pts)
    f = dict(dtype=torch.float32, device="cuda")
    return dict(env=env, pts=pts, cam=cam, q=[y * 64 + x for y, x in PIXELS],
                n=torch.tensor([[0.0, 0.0, 1.0]] * M, **f), v=torch.tensor(cam[None] - pts, **f),
                base=torch.full((M, 3), 0.5, **f), rough=torch.full((M, 1), rough, **f))


def sample_rows(pr, s, N):
    """importance_sample at the plane's pixels as rows of a 48 x 64 image (row q = y W + x)"""
    idx = torch.tensor(pr["q"], device="cuda")
    n = torch.zeros(48 * 64, 3, device="cuda")
    n[:, 2] = 1
    v = torch.zeros(48 * 64, 3, device="cuda")
    v[idx] = pr["v"]
    r = torch.full((48 * 64, 1), float(pr["rough"][0, 0]), device="cuda")
    dirs, areas = importance_sample(n, s, N, v, r)
    return dirs[idx].contiguous(), areas[idx].contiguous()


def shade(pr, dirs, areas, base=None, rough=None):
    M, N = dirs.shape[:2]
    pbr, _ = rendering_equation(pr["base"] if base is None else base, pr["rough"] if rough is None else rough, pr["n"], pr["v"],
                                torch.zeros(M, 16, 3, device="cuda"), FixedLight(pr["env"]), torch.ones(M, N, 1, device="cuda"),
                                dirs, areas)
    return pbr


@pytest.mark.parametrize("rough", [0.12, 0.5, 0.9])
def test_quality_against_the_quadrature_truth(rough, record_property):
    pr = plane_rows(rough)
    s = EnvSampler(FixedLight(pr["env"]), seed=0)
    dirs, areas = sample_rows(pr, s, 32)
    pbr = shade(pr, dirs, areas).double().cpu().numpy()
    env = I.plane_env()
    n = np.array([0.0, 0.0, 1.0])
    est = np.stack([I.estimate(env, p, n, pr["cam"], 0.5, rough, d, a[:, 0])
                    for p, d, a in zip(pr["pts"], dirs.double().cpu().numpy(), areas.double().cpu().numpy())])
    truth = np.stack([I.truth(env, p, n, pr["cam"], 0.5, rough, 600, 1200) for p in pr["pts"]])
    rel = lambda a, b: float(np.linalg.norm(a - b) / np.linalg.norm(b))
    fib = {}
    for NF in (32, 256):
        dF, aF = fibonacci_sphere_sampling(pr["n"], NF, random_rotate=False)
        fib[NF] = rel(shade(pr, dF, aF).double().cpu().numpy(), truth)
    err = rel(pbr, truth)
    record_property("rel_l2_importance_n32", err)
    record_property("rel_l2_fibonacci_n32", fib[32])
    record_property("rel_l2_fibonacci_n256", fib[256])
    print(f"roughness {rough}: importance N=32 {err:.3e}, Fibonacci N=32 {fib[32]:.3e}, N=256 {fib[256]:.3e}")
    assert rel(pbr, est) <= 1e-3                      # the kernel's fp32 estimate of the same samples
    assert err <= 0.15 and err <= 0.5 * fib[32] and err < fib[256]


def test_gradients_are_unbiased():
    """Mean over 64 seeds of dL/dbase_color and dL/droughness (L = sum of pbr) at every pixel of PIXELS against the
    truth's: the integral of L (n.l) / pi, and a central difference of the quadrature in the roughness."""
    rough = 0.5
    pr = plane_rows(rough)
    gb, gr = [], []
    for seed in range(64):
        s = EnvSampler(FixedLight(pr["env"]), seed=seed)
        dirs, areas = sample_rows(pr, s, 32)
        b = pr["base"].clone().requires_grad_()
        r = pr["rough"].clone().requires_grad_()
        shade(pr, dirs, areas, b, r).sum().backward()
        gb.append(b.grad.double().cpu().numpy())
        gr.append(r.grad[:, 0].double().cpu().numpy())
    gb, gr = np.array(gb), np.array(gr)                                        # [64,M,3], [64,M]
    env, n, cam, h = I.plane_env(), np.array([0.0, 0.0, 1.0]), pr["cam"], 1e-3
    for k, p in enumerate(pr["pts"]):
        t_b = I.truth(env, p, n, cam, 1.0, rough, 600, 1200) - I.truth(env, p, n, cam, 0.0, rough, 600, 1200)
        t_r = float((I.truth(env, p, n, cam, 0.5, rough + h, 600, 1200) - I.truth(env, p, n, cam, 0.5, rough - h, 600, 1200)).sum() / (2 * h))
        se_b, se_r = gb[:, k].std(0, ddof=1) / 8, gr[:, k].std(ddof=1) / 8
        print(f"pixel {PIXELS[k]}: dL/dbase {gb[:, k].mean(0)[0]:.5f} truth {t_b[0]:.5f} se {se_b[0]:.5f}; "
              f"dL/drough {gr[:, k].mean():.5f} truth {t_r:.5f} se {se_r:.5f}")
        assert np.all(np.abs(gb[:, k].mean(0) - t_b) <= 3 * se_b + 1e-6 * np.abs(t_b)), PIXELS[k]
        assert abs(gr[:, k].mean() - t_r) <= 3 * se_r + 1e-4 * abs(t_r), PIXELS[k]


def test_deterministic_env_gradient_and_views():
    env_raw = torch.tensor(random_env(16, 32, 9), dtype=torch.float32).cuda()
    T = torch.tensor(rotation(8), dtype=torch.float32).cuda()
    s = EnvSampler(FixedLight(env_raw, T), mix=(0.5, 0.0, 0.5), seed=3)
    P, N = 200, 16
    n, v, r = rows(P, 4)
    dirs, areas = importance_sample(n, s, N)
    base, inc = torch.rand(P, 3, device="cuda"), 0.1 * torch.randn(P, 16, 3, device="cuda")
    vis = torch.ones(P, N, 1, device="cuda")

    def env_grad():
        e = env_raw.clone().requires_grad_()
        pbr, _ = rendering_equation(base, r, n, v, inc, FixedLight(e, T), vis, dirs, areas)
        pbr.sum().backward()
        return e.grad
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        g1, g2 = env_grad(), env_grad()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert bits_equal(g1, g2) and float(g1.abs().sum()) > 0
    vv = torch.stack([v, -v + 0.3])
    pbr_v, _ = rendering_equation_views(base, r, n, vv, inc, FixedLight(env_raw, T), vis, dirs, areas, sampler=s)
    for k in range(2):
        one, _ = rendering_equation(base, r, n, vv[k], inc, FixedLight(env_raw, T), vis, dirs, areas)
        assert bits_equal(pbr_v[k], one)


# ---- per-pixel path -----------------------------------------------------------------------------------------------------
from test_pixel_shading_gpu import gbuffer, rows as img_rows, scene  # noqa: E402


def pixel_rows(c, v, s, N):
    """importance_sample of view v's pixels as rows (row p = y W + x), as the per-pixel kernels sample them"""
    pick = (lambda t: t[v]) if c["normal"].dim() == 4 else (lambda t: t)
    campos = c["campos"][v] if c["campos"].dim() == 2 else c["campos"]
    return importance_sample(img_rows(pick(c["normal"])), s, N, campos[None] - img_rows(pick(c["points"])),
                             img_rows(pick(c["roughness"])))


@pytest.mark.parametrize("H,W,V,masked", [(13, 29, 0, False), (16, 20, 0, True), (9, 11, 3, True)])
def test_trace_pixels_with_sampler_equals_the_rows(H, W, V, masked):
    N = 16
    rt, sc = scene(2000, "shell-v1")
    c = gbuffer(H, W, V, N)
    s = EnvSampler(FixedLight(F.softplus(c["env_raw"][0]), c["rot"][0] if V else c["rot"]), seed=9)
    mask = c["mask"] if masked else None
    T = rt.trace_pixels(c["points"], c["normal"], N, sc["means3D"], sc["inv"], sc["opacity"], sc["normals"], mask=mask,
                        sampler=s, roughness=c["roughness"], campos=c["campos"])
    for v in range(max(V, 1)):
        dirs, _ = pixel_rows(c, v, s, N)
        pts = img_rows(c["points"][v] if V else c["points"])
        ref = rt.trace_visibility(pts[:, None].expand(-1, N, -1), dirs, sc["means3D"], sc["inv"], sc["opacity"],
                                  sc["normals"])["visibility"][..., 0]                       # [HW,N]
        got = (T[v] if V else T).reshape(N, H * W).T.contiguous()
        keep = torch.ones(H * W, dtype=torch.bool, device="cuda") if mask is None else (mask[v] if V else mask).reshape(-1)
        assert bits_equal(got[keep], ref[keep])
        assert torch.all(got[~keep] == 0)


@pytest.mark.parametrize("with_inc,filt,per_view", [(True, False, False), (False, True, False), (True, True, True)])
def test_shade_pixels_with_sampler_equals_the_rows(with_inc, filt, per_view):
    H, W, N = 11, 13, 16
    V = 2 if per_view else 0
    c = gbuffer(H, W, V, N)
    env = F.softplus(c["env_raw"][0])
    tr = c["rot"] if per_view else c["rot"]
    s = EnvSampler(FixedLight(env, c["rot"][0] if per_view else tr), seed=4)
    light = FixedLight(env, tr)
    leaves = {"base_color": c["base_color"].clone().requires_grad_(), "roughness": c["roughness"].clone().requires_grad_(),
              "incidents": c["incidents"].clone().requires_grad_() if with_inc else None}
    e_pix = env.clone().requires_grad_()
    out = shade_pixels(leaves["base_color"], leaves["roughness"], c["normal"], c["points"], c["campos"], c["T"],
                       FixedLight(e_pix, tr), incidents=leaves["incidents"], env_filter=filt, sampler=s)
    loss = sum((out[k] * c["cot"][k]).sum() for k in ("pbr", "diffuse_light", "specular"))
    loss.backward()
    e_row = env.clone().requires_grad_()
    for v in range(max(V, 1)):
        pick = (lambda t: t[v]) if V else (lambda t: t)
        dirs, areas = pixel_rows(c, v, s, N)
        b = img_rows(pick(c["base_color"])).requires_grad_()
        r = img_rows(pick(c["roughness"])).requires_grad_()
        inc = (img_rows(pick(c["incidents"])) if with_inc else torch.zeros(H * W, 48, device="cuda")).reshape(-1, 16, 3).requires_grad_()
        campos = c["campos"][v] if V else c["campos"]
        pbr, extra = rendering_equation(b, r, img_rows(pick(c["normal"])), campos[None] - img_rows(pick(c["points"])), inc,
                                        FixedLight(e_row, tr[v] if per_view else tr), img_rows(pick(c["T"]))[..., None],
                                        dirs, areas, env_filter=filt)
        ref = {"pbr": pbr, "diffuse_light": extra["diffuse_light"], "specular": extra["specular"]}
        for k in ref:
            assert bits_equal(pick(out[k]), ref[k].T.reshape(3, H, W)), k
        sum((ref[k].T.reshape(3, H, W) * pick(c["cot"][k])).sum() for k in ref).backward()
        rel = lambda x, y: float((x.double() - y.double()).norm() / (y.double().norm() + 1e-30))
        assert rel(img_rows(pick(leaves["base_color"].grad)), b.grad) <= 1e-5
        assert rel(img_rows(pick(leaves["roughness"].grad)), r.grad) <= 1e-5
        if with_inc:
            assert rel(img_rows(pick(leaves["incidents"].grad)).reshape(-1, 16, 3), inc.grad) <= 1e-5
    assert rel(e_pix.grad, e_row.grad) <= 1e-5


def test_shade_pixels_with_sampler_deterministic_and_refusals():
    H, W, N = 9, 10, 8
    c = gbuffer(H, W, 0, N)
    env = F.softplus(c["env_raw"][0])
    s = EnvSampler(FixedLight(env), seed=1)

    def env_grad():
        e = env.clone().requires_grad_()
        out = shade_pixels(c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], FixedLight(e),
                           sampler=s)
        out["pbr"].sum().backward()
        return e.grad
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        g1, g2 = env_grad(), env_grad()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert bits_equal(g1, g2)
    with pytest.raises(ValueError, match="transform"):
        shade_pixels(c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], FixedLight(env, c["rot"]),
                     sampler=s)
    with pytest.raises(ValueError, match="env is"):
        shade_pixels(c["base_color"], c["roughness"], c["normal"], c["points"], c["campos"], c["T"], FixedLight(env[:8]),
                     sampler=s)
    rt, sc = scene(500, "shell-v1")
    with pytest.raises(ValueError, match="roughness and campos"):
        rt.trace_pixels(c["points"], c["normal"], N, sc["means3D"], sc["inv"], sc["opacity"], sc["normals"], sampler=s)


@pytest.mark.parametrize("rough", [0.12, 0.5, 0.9])
def test_shade_pixels_quality_against_the_quadrature_truth(rough, record_property):
    H, W, N = 48, 64, 32
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1.4, 1.4, W), indexing="ij")
    pts = torch.stack([xs, ys, torch.zeros_like(xs)]).cuda()
    nrm = torch.tensor([0.0, 0.0, 1.0]).view(3, 1, 1).expand(3, H, W).contiguous().cuda()
    base = torch.full((3, H, W), 0.5).cuda()
    rg = torch.full((1, H, W), rough).cuda()
    campos = torch.tensor(I.plane_pixel()[2], dtype=torch.float32).cuda()
    env = torch.tensor(I.plane_env(), dtype=torch.float32).cuda()
    s = EnvSampler(FixedLight(env), seed=0)
    shade = lambda n_s, smp: shade_pixels(base, rg, nrm, pts, campos, torch.ones((n_s, H, W), device="cuda"), FixedLight(env),
                                          sampler=smp)["pbr"]
    idx = [y * W + x for y, x in PIXELS]
    at = lambda img: img.reshape(3, -1)[:, idx].T.double().cpu().numpy()
    got = at(shade(N, s))
    dirs, areas = importance_sample(img_rows(nrm), s, N, campos[None] - img_rows(pts), img_rows(rg))
    n = np.array([0.0, 0.0, 1.0])
    ps = img_rows(pts).double().cpu().numpy()[idx]
    est = np.stack([I.estimate(I.plane_env(), p, n, I.plane_pixel()[2], 0.5, rough, dirs[q].double().cpu().numpy(),
                               areas[q, :, 0].double().cpu().numpy()) for p, q in zip(ps, idx)])
    truth = np.stack([I.truth(I.plane_env(), p, n, I.plane_pixel()[2], 0.5, rough, 600, 1200) for p in ps])
    rel = lambda x, y: float(np.linalg.norm(x - y) / np.linalg.norm(y))
    err, fib32, fib256 = rel(got, truth), rel(at(shade(32, None)), truth), rel(at(shade(256, None)), truth)
    record_property("rel_l2_shade_pixels_importance_n32", err)
    record_property("rel_l2_shade_pixels_fibonacci_n32", fib32)
    record_property("rel_l2_shade_pixels_fibonacci_n256", fib256)
    print(f"shade_pixels roughness {rough}: importance N=32 {err:.3e}, Fibonacci N=32 {fib32:.3e}, N=256 {fib256:.3e}")
    assert rel(got, est) <= 1e-3
    assert err <= 0.15 and err <= 0.5 * fib32 and err < fib256
