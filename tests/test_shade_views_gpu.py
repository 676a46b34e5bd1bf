"""Several views in one shading call (shading.rendering_equation_views) against one-view `rendering_equation` calls on
the same inputs: forward outputs bit for bit, leaf gradients equal to the sum of the one-view gradients, per-view
viewdir gradients equal to the one-view ones, agreement with the PyTorch oracle, the deterministic mode, and a
V-view stage-2 step (shading, feature pack, several-view rasterizer, unpremultiply, L1 losses)."""
import pytest
import torch
import torch.nn.functional as F

from helpers import npy, rel_l2, shading_case
from relightable3dgaussian_b200 import shading
from relightable3dgaussian_b200.shading import _RenderEquation, rendering_equation, rendering_equation_views

pytestmark = pytest.mark.gpu
LEAVES = ("base_color", "roughness", "incidents")


class SoftplusLight:            # duck-types DirectLightMap (get_env property)
    def __init__(self, env_raw):
        self.env = env_raw

    @property
    def get_env(self):
        return F.softplus(self.env)


class FixedLight:               # duck-types EnvLight (envmap + transform)
    def __init__(self, envmap, transform=None):
        self.envmap, self.transform = envmap, transform


def views_case(P, N, He, V, seed=3):
    """shading_case plus V random unit view directions, V random rotations and per-view cotangents."""
    c = {k: v.cuda() for k, v in shading_case(P, N, He, seed).items()}
    g = torch.Generator().manual_seed(900 + seed)
    c["viewdirs_v"] = F.normalize(torch.randn(V, P, 3, generator=g), dim=-1).cuda()
    c["rot_v"] = torch.linalg.qr(torch.randn(V, 3, 3, generator=g, dtype=torch.float64))[0].float().cuda()
    for k in ("pbr", "diffuse", "specular"):
        c["vcot_" + k] = torch.randn(V, P, 3, generator=g).cuda()
    return c


def light_of(kind, c, env_raw, v=None):
    if kind == "softplus":
        return SoftplusLight(env_raw)
    tex = F.softplus(env_raw)[0]
    if kind == "fixed":
        return FixedLight(tex, c["rot_v"][0])
    return FixedLight(tex, c["rot_v"] if v is None else c["rot_v"][v])     # per-view transforms


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ---- 1. forward: every view bit for bit equal to a one-view call ------------------------------------------------------
# V = 9 and 64 cross the 8-view launch chunks; P = 1, 5, 33 leave groups idle; N = 3, 7 are fewer samples than lanes;
# He = 16 keeps the texture in shared memory, 128 reads it from global memory
FWD_CASES = [(1, 1, 3, 16), (2, 5, 7, 16), (3, 33, 64, 128), (8, 30_000, 64, 16), (9, 33, 7, 128), (9, 5, 3, 16),
             (64, 33, 3, 16), (8, 1, 64, 128), (3, 30_000, 7, 128), (2, 1, 3, 128)]


@pytest.mark.parametrize("light", ["softplus", "fixed", "per_view"])
@pytest.mark.parametrize("V,P,N,He", FWD_CASES)
def test_forward_bitwise_against_one_view_calls(V, P, N, He, light):
    c = views_case(P, N, He, V)
    with torch.no_grad():
        for means in (False, True):
            pbr, ex = rendering_equation_views(c["base_color"], c["roughness"], c["normals"], c["viewdirs_v"], c["incidents"],
                                               light_of(light, c, c["env_raw"]), c["visibility"], c["incident_dirs"],
                                               c["incident_areas"], means=means)
            assert ex["incident_dirs"] is c["incident_dirs"] and ex["incident_visibility"] is c["visibility"]
            assert set(ex) == {"incident_dirs", "incident_visibility", "diffuse_light", "specular"} | (set(shading._MEANS) if means else set())
            for v in range(V):
                lt = light_of(light, c, c["env_raw"], v)
                tex, tr = (lt.get_env[0], None) if light == "softplus" else (lt.envmap, lt.transform)
                one = _RenderEquation.apply(c["base_color"], c["roughness"], c["viewdirs_v"][v], c["incidents"], tex, c["normals"],
                                            c["visibility"], c["incident_dirs"], c["incident_areas"], tr, means)
                got = [pbr[v], ex["diffuse_light"][v], ex["specular"][v]] + ([ex[k][v] for k in shading._MEANS] if means else [])
                for k, (a, b) in enumerate(zip(got, one)):
                    assert bits_equal(a, b), (v, k, means, (a - b).abs().max().item())


# ---- 2. backward: the sum of one-view backward calls --------------------------------------------------------------------
def _views_grads(c, light_kind="softplus"):
    leaves = {k: c[k].clone().requires_grad_(True) for k in LEAVES}
    vd = c["viewdirs_v"].clone().requires_grad_(True)
    env_raw = c["env_raw"].clone().requires_grad_(True)
    pbr, ex = rendering_equation_views(leaves["base_color"], leaves["roughness"], c["normals"], vd, leaves["incidents"],
                                       light_of(light_kind, c, env_raw), c["visibility"], c["incident_dirs"], c["incident_areas"])
    ((pbr * c["vcot_pbr"]).sum() + (ex["diffuse_light"] * c["vcot_diffuse"]).sum()
     + (ex["specular"] * c["vcot_specular"]).sum()).backward()
    out = {k: v.grad for k, v in leaves.items()}
    out.update(env_raw=env_raw.grad, viewdirs=vd.grad)
    return out


def _one_view_grads_summed(c, light_kind="softplus"):
    V = c["viewdirs_v"].shape[0]
    tot, dviews = {}, []
    for v in range(V):
        leaves = {k: c[k].clone().requires_grad_(True) for k in LEAVES}
        vd = c["viewdirs_v"][v].clone().requires_grad_(True)
        env_raw = c["env_raw"].clone().requires_grad_(True)
        pbr, ex = rendering_equation(leaves["base_color"], leaves["roughness"], c["normals"], vd, leaves["incidents"],
                                     light_of(light_kind, c, env_raw), c["visibility"], c["incident_dirs"], c["incident_areas"])
        ((pbr * c["vcot_pbr"][v]).sum() + (ex["diffuse_light"] * c["vcot_diffuse"][v]).sum()
         + (ex["specular"] * c["vcot_specular"][v]).sum()).backward()
        for k, t in list({k: l.grad for k, l in leaves.items()}.items()) + [("env_raw", env_raw.grad)]:
            tot[k] = tot.get(k, 0) + t.double()
        dviews.append(vd.grad)
    tot["viewdirs"] = torch.stack(dviews)
    return tot


@pytest.mark.parametrize("V,P,N,He,light", [(4, 30_000, 32, 16, "softplus"), (9, 3_000, 64, 16, "fixed"),
                                             (3, 2_000, 24, 128, "softplus"), (2, 5, 7, 24, "fixed"), (1, 33, 8, 16, "softplus")])
def test_backward_equals_sum_of_one_view_calls(V, P, N, He, light):
    c = views_case(P, N, He, V)
    got, ref = _views_grads(c, light), _one_view_grads_summed(c, light)
    errs = {k: rel_l2(npy(got[k]), npy(ref[k])) for k in (*LEAVES, "env_raw")}
    errs_v = [rel_l2(npy(got["viewdirs"][v]), npy(ref["viewdirs"][v])) for v in range(V)]
    print(f"\n[shade_views bwd] V={V} P={P} N={N} He={He} {light}: "
          + " ".join(f"{k}={e:.2e}" for k, e in errs.items()) + f" viewdirs_max={max(errs_v):.2e}")
    for k, e in errs.items():
        assert e <= 1e-5, (k, e)
    assert max(errs_v) <= 1e-6, errs_v


# ---- 3. against the PyTorch oracle, per view and summed -----------------------------------------------------------------
@pytest.mark.parametrize("V,P,N,He,fixed", [(4, 5_000, 40, 16, False), (3, 2_000, 24, 128, True), (9, 33, 8, 16, True)])
def test_against_pytorch_oracle(V, P, N, He, fixed):
    from oracle import oracle_shading as osh
    c = views_case(P, N, He, V)
    got = _views_grads(c, "fixed" if fixed else "softplus")
    tot, outs = {}, []
    for v in range(V):
        leaves = {k: c[k].clone().requires_grad_(True) for k in LEAVES}
        vd = c["viewdirs_v"][v].clone().requires_grad_(True)
        env_raw = c["env_raw"].clone().requires_grad_(True)
        pbr, ex = osh.rendering_equation(leaves["base_color"], leaves["roughness"], c["normals"], vd, leaves["incidents"],
                                         F.softplus(env_raw)[0], c["visibility"], c["incident_dirs"], c["incident_areas"],
                                         transform=c["rot_v"][0] if fixed else None)
        ((pbr * c["vcot_pbr"][v]).sum() + (ex["diffuse_light"] * c["vcot_diffuse"][v]).sum()
         + (ex["specular"] * c["vcot_specular"][v]).sum()).backward()
        for k, t in list({k: l.grad for k, l in leaves.items()}.items()) + [("env_raw", env_raw.grad), ("viewdirs", vd.grad)]:
            tot.setdefault(k, []).append(t)
        outs.append((pbr.detach(), ex["diffuse_light"].detach(), ex["specular"].detach()))
    with torch.no_grad():
        pbr, ex = rendering_equation_views(c["base_color"], c["roughness"], c["normals"], c["viewdirs_v"], c["incidents"],
                                           light_of("fixed" if fixed else "softplus", c, c["env_raw"]), c["visibility"],
                                           c["incident_dirs"], c["incident_areas"])
    for v in range(V):
        for a, b in zip((pbr[v], ex["diffuse_light"][v], ex["specular"][v]), outs[v]):
            torch.testing.assert_close(a, b, rtol=5e-4, atol=1e-4)
    for k in (*LEAVES, "env_raw"):
        assert rel_l2(npy(got[k]), npy(sum(t.double() for t in tot[k]))) < 1e-3, k
    assert rel_l2(npy(got["viewdirs"]), npy(torch.stack(tot["viewdirs"]))) < 1e-3


# ---- 4. deterministic mode ----------------------------------------------------------------------------------------------
@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("V,P,N,He", [(4, 20_000, 32, 16), (9, 3_000, 24, 128)])
def test_deterministic_mode_is_bitwise_reproducible(V, P, N, He, det_mode):
    c = views_case(P, N, He, V)
    a, b = _views_grads(c), _views_grads(c)
    for k in a:
        assert bits_equal(a[k], b[k]), k
    torch.use_deterministic_algorithms(False)
    d = _views_grads(c)
    for k in a:
        assert rel_l2(npy(a[k]), npy(d[k])) <= 1e-5, (k, rel_l2(npy(a[k]), npy(d[k])))


# ---- 5. P = 0 -------------------------------------------------------------------------------------------------------------
def test_empty_gaussian_set():
    c = views_case(0, 8, 16, 3)
    vd = c["viewdirs_v"].clone().requires_grad_(True)
    env_raw = c["env_raw"].clone().requires_grad_(True)
    bc = c["base_color"].clone().requires_grad_(True)
    pbr, ex = rendering_equation_views(bc, c["roughness"], c["normals"], vd, c["incidents"], SoftplusLight(env_raw),
                                       c["visibility"], c["incident_dirs"], c["incident_areas"], means=True)
    assert pbr.shape == (3, 0, 3) and ex["specular"].shape == (3, 0, 3) and ex["mean_incident_visibility"].shape == (3, 0, 1)
    (pbr.sum() + ex["diffuse_light"].sum()).backward()
    assert env_raw.grad is not None and not env_raw.grad.any()
    assert vd.grad.shape == (3, 0, 3) and bc.grad.shape == (0, 3)
    # one view: the same node, forward and backward
    vd1 = c["viewdirs_v"][0].clone().requires_grad_(True)
    env_raw.grad = bc.grad = None
    pbr, ex = rendering_equation(bc, c["roughness"], c["normals"], vd1, c["incidents"], SoftplusLight(env_raw),
                                 c["visibility"], c["incident_dirs"], c["incident_areas"])
    assert pbr.shape == (0, 3) and ex["specular"].shape == (0, 3) and ex["incident_lights"].shape == (0, 8, 3)
    (pbr.sum() + ex["diffuse_light"].sum()).backward()
    assert env_raw.grad is not None and not env_raw.grad.any()
    assert vd1.grad.shape == (0, 3) and bc.grad.shape == (0, 3)


# ---- 6. a V-view stage-2 step against V one-view steps --------------------------------------------------------------------
def test_stage2_step_of_four_views_against_one_view_steps():
    from relightable3dgaussian_b200 import synth
    from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, pack_features,
                                                        rasterize_views, unpremultiply)
    V, P, N, W, H = 4, 3_000, 32, 96, 72
    sc = synth.make_scene(P, "shell-v1", 0, 0)
    sh = shading_case(P, N, 16, seed=5)
    cams = [synth.make_camera(k, W, H) for k in range(V)]
    bg = torch.tensor([0.1, 0.2, 0.3]).cuda()
    settings = [GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, bg, 1.0, c.viewmatrix.cuda(),
                                              c.projmatrix.cuda(), 3, c.campos.cuda(), False, True, True, False) for c in cams]
    g = torch.Generator().manual_seed(11)
    gts = [torch.rand(3, H, W, generator=g).cuda() for _ in range(V)]
    init = dict(means3D=sc.means3D, opacities=sc.opacities, shs=sc.shs, scales=sc.scales, rotations=sc.rotations,
                normal=sc.normals, base_color=sh["base_color"], roughness=sh["roughness"], incidents=sh["incidents"],
                env=sh["env_raw"])
    fixed = {k: sh[k].cuda() for k in ("visibility", "incident_dirs", "incident_areas")}

    def step(batched):
        m = {k: v.cuda().contiguous().requires_grad_(True) for k, v in init.items()}
        nrm = F.normalize(m["normal"], dim=-1)
        vis_mean = fixed["visibility"].mean(1)
        viewdirs = torch.stack([F.normalize(s.campos - m["means3D"], dim=-1) for s in settings])
        light = SoftplusLight(m["env"])
        if batched:
            pbr, ex = rendering_equation_views(m["base_color"], m["roughness"], nrm.detach(), viewdirs, m["incidents"], light,
                                               fixed["visibility"], fixed["incident_dirs"], fixed["incident_areas"])
        else:
            res = [rendering_equation(m["base_color"], m["roughness"], nrm.detach(), viewdirs[v], m["incidents"], light,
                                      fixed["visibility"], fixed["incident_dirs"], fixed["incident_areas"]) for v in range(V)]
            pbr = torch.stack([r[0] for r in res])
            ex = {"diffuse_light": torch.stack([r[1]["diffuse_light"] for r in res])}
        feats = [pack_features([pbr[v], nrm, m["base_color"], m["roughness"], ex["diffuse_light"][v], vis_mean],
                               means3D=m["means3D"], viewmatrix=settings[v].viewmatrix) for v in range(V)]
        geo = dict(shs=m["shs"], scales=m["scales"], rotations=m["rotations"])
        if batched:
            out = rasterize_views(m["means3D"], torch.zeros(V, P, 3, device="cuda"), m["opacities"], settings=settings,
                                  features=torch.stack(feats), **geo)
            views = [(out[2][v], out[3][v], out[5][v], out[1][v]) for v in range(V)]
        else:
            views = []
            for v in range(V):
                o = GaussianRasterizer(settings[v])(m["means3D"], torch.zeros(P, 3, device="cuda"), m["opacities"],
                                                    features=feats[v], **geo)
                views.append((o[2], o[3], o[5], o[1]))
        loss = 0
        for v, (color, opacity, feature, n_contrib) in enumerate(views):
            feature = unpremultiply(feature, opacity, n_contrib)
            pbr_img = feature[2:5] * opacity + (1 - opacity) * bg[:, None, None]
            loss = loss + (color - gts[v]).abs().mean() + (pbr_img - gts[v]).abs().mean()
        loss.backward()
        return {k: t.grad for k, t in m.items()}

    got, ref = step(True), step(False)
    for k in init:
        if ref[k] is None:
            assert got[k] is None, k
            continue
        e = rel_l2(npy(got[k]), npy(ref[k]))
        print(f"[shade_views stage2] {k}: {e:.2e}")
        assert e <= 1e-5, (k, e)
