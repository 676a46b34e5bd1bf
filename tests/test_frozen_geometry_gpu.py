"""Appearance-only rasterizer backward (frozen geometry): when no geometry input requires grad, the backward computes only
the features / colors_precomp / shs gradients.  The same forward, differentiated with every input requiring grad and with
only the appearance inputs requiring grad, gives the same appearance gradients: bitwise in deterministic mode, within
float-atomic spread otherwise, +0 on rows no pixel composited, with fewer library launches."""
import pytest
import torch
import torch.nn.functional as F

from helpers import npy, rel_l2, shading_case
from relightable3dgaussian_b200 import _lib, synth
from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, pack_features,
                                                    rasterize_views, unpremultiply)
from relightable3dgaussian_b200.shading import rendering_equation

pytestmark = pytest.mark.gpu

P, W, H = 3_000, 96, 72
GEOMETRY = ("means3D", "opacities", "scales", "rotations")
APPEARANCE = ("features", "shs", "colors_precomp")


@pytest.fixture(params=[False, True], ids=["default", "det"])
def det(request):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(request.param)
    yield request.param
    torch.use_deterministic_algorithms(prev)


def make_inputs(S, colors, views, seed=0):
    """Leaves (CPU), settings of V views, the per-view cotangents and the rows that can never composite (opacity 1e-4:
    alpha < 1/255 at every pixel).  views: "one" (GaussianRasterizer), "shared3" / "perview3" (rasterize_views)."""
    V = 1 if views == "one" else 3
    sc = synth.make_scene(P, seed=seed, S=S)
    g = torch.Generator().manual_seed(seed + 1)
    dead = torch.zeros(P, dtype=torch.bool)
    dead[::10] = True
    opac = sc.opacities.clone()
    opac[dead] = 1e-4
    leaves = dict(means3D=sc.means3D, opacities=opac, scales=sc.scales, rotations=sc.rotations)
    if colors:
        leaves["colors_precomp"] = torch.rand(P, 3, generator=g)
    else:
        leaves["shs"] = sc.shs
    if S > 0:
        leaves["features"] = (torch.stack([sc.features + 0.1 * k for k in range(V)]) if views == "perview3"
                              else sc.features)
    cams = [synth.make_camera(k, W, H, center_shift=(k % 2 == 1)) for k in range(V)]
    cot = [dict(color=torch.randn(3, H, W, generator=g), opacity=torch.randn(1, H, W, generator=g),
                depth=torch.randn(1, H, W, generator=g) * 0.1, feature=torch.randn(S, H, W, generator=g))
           for _ in range(V)]
    return leaves, cams, cot, dead


def run(leaves, cams, cot, views, grad, camera_grad=False):
    """Forward + backward with the leaves in `grad` requiring grad (means2D is one of them by name); returns the leaves'
    gradients and the library launches of the backward."""
    lib = _lib.load()
    m = {k: v.cuda().contiguous().requires_grad_(k in grad) for k, v in leaves.items()}
    mats = [{k: getattr(c, k).cuda().requires_grad_(camera_grad or k in grad) for k in ("viewmatrix", "projmatrix", "campos")}
            for c in cams]
    bg = torch.tensor([0.1, 0.4, 0.7]).cuda()
    settings = [GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, bg, 1.0, mt["viewmatrix"],
                                              mt["projmatrix"], 3, mt["campos"], False, True, True, False)
                for c, mt in zip(cams, mats)]
    kw = {k: m[k] for k in ("shs", "colors_precomp", "scales", "rotations", "features") if k in m}
    V = len(cams)
    if views == "one":
        means2D = torch.zeros(P, 3, device="cuda", requires_grad="means2D" in grad)
        out = GaussianRasterizer(settings[0])(m["means3D"], means2D, m["opacities"], **kw)
        imgs = [(out[2], out[3], out[4], out[5])]
    else:
        means2D = torch.zeros(V, P, 3, device="cuda", requires_grad="means2D" in grad)
        out = rasterize_views(m["means3D"], means2D, m["opacities"], settings=settings, **kw)
        imgs = [(out[2][v], out[3][v], out[4][v], out[5][v]) for v in range(V)]
    loss = 0
    for (color, opacity, depth, feature), c in zip(imgs, cot):
        loss = loss + (color * c["color"].cuda()).sum() + (opacity * c["opacity"].cuda()).sum()
        loss = loss + (depth * c["depth"].cuda()).sum() + (feature * c["feature"].cuda()).sum()
    torch.cuda.synchronize()
    n0 = lib.r3dg_launch_count()
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: t.grad for k, t in m.items()}
    grads["means2D"] = means2D.grad
    return grads, lib.r3dg_launch_count() - n0


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("views", ["one", "shared3", "perview3"])
@pytest.mark.parametrize("colors", [False, True], ids=["sh3", "colors"])
@pytest.mark.parametrize("S", [0, 5, 16, 24])
def test_appearance_grads_equal_full_backward(S, colors, views, det):
    leaves, cams, cot, dead = make_inputs(S, colors, views)
    V = len(cams)
    full, n_full = run(leaves, cams, cot, views, grad=set(leaves) | {"means2D"}, camera_grad=True)
    app_in = {k for k in leaves if k in APPEARANCE}
    app, n_app = run(leaves, cams, cot, views, grad=app_in)
    for k in app_in:
        a, f = app[k], full[k]
        assert a is not None and a.shape == f.shape, k
        if det:
            assert bits_equal(a, f), k
        else:
            e = rel_l2(npy(a), npy(f))
            assert e <= 1e-6, (k, e)
        rows = a[:, dead] if k == "features" and views == "perview3" else a[dead]      # [V,P,S] per-view features
        assert torch.all(rows == 0) and not torch.any(torch.signbit(rows)), k
    for k in GEOMETRY + ("means2D",):
        assert app[k] is None, k
    # full: zero rows, CTA order, composite, a projection backward per view, camera sums (+ the SH rebuild of V views);
    # appearance: zero rows, CTA order, composite, one launch for the colour / feature / SH outputs (+ the SH rebuild)
    rebuild = 1 if V > 1 and not colors else 0
    assert n_full == 3 + V + 1 + rebuild, n_full
    assert n_app == 4 + rebuild, n_app
    assert n_app < n_full


@pytest.mark.parametrize("views", ["one", "shared3"])
@pytest.mark.parametrize("which", ["means2D", "viewmatrix", "campos"])
def test_one_geometry_input_takes_the_full_backward(which, views, det):
    """A single geometry input that requires grad launches exactly what the full backward launches, and the appearance
    gradients are those of the full backward."""
    leaves, cams, cot, _ = make_inputs(5, False, views)
    V = len(cams)
    camera = which != "means2D"
    full, n_full = run(leaves, cams, cot, views, grad=set(leaves) | {"means2D"}, camera_grad=camera)
    one, n_one = run(leaves, cams, cot, views, grad={"features", "shs", which})
    assert n_one == n_full == 3 + V + (1 if camera else 0) + (1 if V > 1 else 0), (n_one, n_full)
    for k in ("features", "shs"):
        if det:
            assert bits_equal(one[k], full[k]), k
        else:
            assert rel_l2(npy(one[k]), npy(full[k])) <= 1e-6, k
    if which == "means2D":
        assert one["means2D"] is not None and (bits_equal(one["means2D"], full["means2D"]) or not det)


def test_surface_grads_under_frozen_geometry_take_the_appearance_backward():
    """surface_grads=True with frozen geometry: the normal and surface_xyz cotangents reach nothing, and the backward is
    the appearance-only one."""
    leaves, cams, cot, _ = make_inputs(5, False, "one")
    lib = _lib.load()
    c = cams[0]
    bg = torch.tensor([0.1, 0.4, 0.7]).cuda()
    rs = GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, bg, 1.0, c.viewmatrix.cuda(),
                                       c.projmatrix.cuda(), 3, c.campos.cuda(), False, True, True, False)
    feats = leaves["features"].cuda().requires_grad_(True)
    out = GaussianRasterizer(rs, surface_grads=True)(leaves["means3D"].cuda(), torch.zeros(P, 3, device="cuda"),
                                                     leaves["opacities"].cuda(), shs=leaves["shs"].cuda(),
                                                     scales=leaves["scales"].cuda(), rotations=leaves["rotations"].cuda(),
                                                     features=feats)
    loss = (out[5] * cot[0]["feature"].cuda()).sum() + out[6].square().sum() + out[7].sum()
    torch.cuda.synchronize()
    n0 = lib.r3dg_launch_count()
    loss.backward()
    torch.cuda.synchronize()
    assert lib.r3dg_launch_count() - n0 == 4
    ref, _ = run(leaves, cams, cot, "one", grad={"features"})
    # the same features cotangent: the surface terms add nothing to dL/dfeatures
    assert rel_l2(npy(feats.grad), npy(ref["features"])) <= 1e-6


def test_stage2_step_with_frozen_geometry(det):
    """A stage-2 step (shade, pack_features, rasterize, unpremultiply, L1) with frozen geometry gives the base_color,
    roughness, incidents and env gradients of the same step with the geometry requiring grad."""
    N = 32
    sc = synth.make_scene(P, "shell-v1", 0, 0)
    sh = shading_case(P, N, 16, seed=5)
    c = synth.make_camera(1, W, H)
    bg = torch.tensor([0.1, 0.2, 0.3]).cuda()
    rs = GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, bg, 1.0, c.viewmatrix.cuda(),
                                       c.projmatrix.cuda(), 3, c.campos.cuda(), False, True, True, False)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(11)).cuda()
    init = dict(means3D=sc.means3D, opacities=sc.opacities, shs=sc.shs, scales=sc.scales, rotations=sc.rotations,
                normal=sc.normals, base_color=sh["base_color"], roughness=sh["roughness"], incidents=sh["incidents"],
                env=sh["env_raw"])
    learnt = ("base_color", "roughness", "incidents", "env")
    fixed = {k: sh[k].cuda() for k in ("visibility", "incident_dirs", "incident_areas")}

    class Light:
        def __init__(self, env_raw):
            self.env = env_raw

        @property
        def get_env(self):
            return F.softplus(self.env)

    def step(frozen):
        m = {k: v.cuda().contiguous().requires_grad_(not frozen or k in learnt) for k, v in init.items()}
        nrm = F.normalize(m["normal"], dim=-1)
        vis_mean = fixed["visibility"].mean(1)
        viewdirs = F.normalize(rs.campos - m["means3D"], dim=-1)
        pbr, ex = rendering_equation(m["base_color"], m["roughness"], nrm.detach(), viewdirs, m["incidents"],
                                     Light(m["env"]), fixed["visibility"], fixed["incident_dirs"], fixed["incident_areas"])
        feats = pack_features([pbr, nrm, m["base_color"], m["roughness"], ex["diffuse_light"], vis_mean],
                              means3D=m["means3D"], viewmatrix=rs.viewmatrix)
        means2D = torch.zeros(P, 3, device="cuda", requires_grad=not frozen)
        out = GaussianRasterizer(rs)(m["means3D"], means2D, m["opacities"], shs=m["shs"], scales=m["scales"],
                                     rotations=m["rotations"], features=feats)
        feature = unpremultiply(out[5], out[3], out[1])
        pbr_img = feature[2:5] * out[3] + (1 - out[3]) * bg[:, None, None]
        loss = (out[2] - gt).abs().mean() + (pbr_img - gt).abs().mean()
        loss.backward()
        return {k: t.grad for k, t in m.items()}

    frozen, full = step(True), step(False)
    for k in init:
        if k not in learnt:
            assert frozen[k] is None, k
            continue
        assert frozen[k] is not None, k
        if det:
            assert bits_equal(frozen[k], full[k]), k
        else:
            e = rel_l2(npy(frozen[k]), npy(full[k]))
            assert e <= 1e-6, (k, e)
