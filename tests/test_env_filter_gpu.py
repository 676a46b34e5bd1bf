"""The shading step's filtered environment lookup on the GPU against its fp64 oracle (tests/envfilter64.py): the pyramid
build, the forward and backward of one view and several views, both light kinds, every r3dg_tune shading variant, the
exact fallback at footprints below a texel, the deterministic mode, the process default and the refusals."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import envfilter64 as ef
from helpers import npy, rel_l2, shading_case
from relightable3dgaussian_b200 import _lib, shading
from relightable3dgaussian_b200.shading import rendering_equation, rendering_equation_views

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


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def case(P, N, He, seed=3, V=None):
    c = {k: v.cuda() for k, v in shading_case(P, N, He, seed).items()}
    g = torch.Generator().manual_seed(77 + seed)
    c["rot"] = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))[0].float().cuda()
    if V:
        c["viewdirs_v"] = F.normalize(torch.randn(V, P, 3, generator=g), dim=-1).cuda()
        c["rot_v"] = torch.linalg.qr(torch.randn(V, 3, 3, generator=g, dtype=torch.float64))[0].float().cuda()
        for k in ("pbr", "diffuse", "specular"):
            c["vcot_" + k] = torch.randn(V, P, 3, generator=g).cuda()
    return c


def light(kind, c, env_raw):
    if kind == "softplus":
        return SoftplusLight(env_raw)
    return FixedLight(F.softplus(env_raw)[0], c["rot"] if kind == "fixed_rot" else None)


# ---- 1. the pyramid build ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("He,We", [(1000, 2000), (512, 1024), (250, 500), (16, 32), (2, 2), (1, 8)])
def test_pyramid_build_against_oracle(He, We):
    lib = _lib.load()
    sizes = ef.level_sizes(He, We)
    assert lib.r3dg_env_pyramid_levels(He, We) == len(sizes)
    assert lib.r3dg_env_pyramid_floats(He, We) == 3 * sum(h * w for h, w in sizes)
    g = torch.Generator().manual_seed(He + We)
    env = (torch.rand(He, We, 3, generator=g) * 4 + 0.05).cuda()
    pyr = torch.empty(lib.r3dg_env_pyramid_floats(He, We), device="cuda")
    again = torch.empty_like(pyr)
    for out in (pyr, again):
        _lib.call("r3dg_env_pyramid_build", env.device, env.data_ptr(), He, We, out.data_ptr())
    assert bits_equal(pyr, again)
    ref = ef.pyramid(env.cpu().double())
    off = 0
    for lv, (h, w) in zip(ref, sizes):
        got = pyr[off:off + 3 * h * w].view(h, w, 3).cpu().double()
        off += 3 * h * w
        err = ((got - lv).abs() / lv.abs()).max().item()
        assert err <= 1e-6, ((h, w), err)


def test_pyramid_of_a_constant_env_is_that_constant():
    env = torch.full((512, 1024, 3), 0.7315, device="cuda")
    pyr = shading.env_pyramid(env)
    assert torch.equal(pyr, torch.full_like(pyr, 0.7315))


# ---- 2. forward against the fp64 oracle ---------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["softplus", "fixed", "fixed_rot"])
@pytest.mark.parametrize("P,N,He", [(3_000, 64, 16), (2_000, 64, 512)])
def test_forward_against_oracle(P, N, He, kind):
    c = case(P, N, He)
    with torch.no_grad():
        lt = light(kind, c, c["env_raw"])
        pbr, ex = rendering_equation(c["base_color"], c["roughness"], c["normals"], c["viewdirs"], c["incidents"], lt,
                                     c["visibility"], c["incident_dirs"], c["incident_areas"], env_filter=True)
        _, exm = rendering_equation_views(c["base_color"], c["roughness"], c["normals"], c["viewdirs"][None], c["incidents"], lt,
                                          c["visibility"], c["incident_dirs"], c["incident_areas"], means=True, env_filter=True)
    tex = F.softplus(c["env_raw"])[0].cpu()
    ref, rex = ef.rendering_equation(*[c[k].cpu() for k in ("base_color", "roughness", "normals", "viewdirs", "incidents")],
                                     tex, *[c[k].cpu() for k in ("visibility", "incident_dirs", "incident_areas")],
                                     transform=c["rot"].cpu() if kind == "fixed_rot" else None)
    pairs = [(pbr, ref), (ex["diffuse_light"], rex["diffuse_light"]), (ex["specular"], rex["specular"])]
    pairs += [(ex[k], rex[k]) for k in ("incident_lights", "local_incident_lights", "global_incident_lights")]
    pairs += [(exm["mean_incident_lights"][0], rex["incident_lights"].mean(1)),
              (exm["mean_local_incident_lights"][0], rex["local_incident_lights"].mean(1)),
              (exm["mean_global_incident_lights"][0], rex["global_incident_lights"].mean(1)),
              (exm["mean_incident_visibility"][0], c["visibility"].cpu().double().mean(1))]
    for k, (a, b) in enumerate(pairs):
        torch.testing.assert_close(a.cpu().double(), b, rtol=5e-4, atol=1e-4, msg=f"output {k}")
    off = rendering_equation(c["base_color"], c["roughness"], c["normals"], c["viewdirs"], c["incidents"], lt,
                             c["visibility"], c["incident_dirs"], c["incident_areas"], env_filter=False)[0]
    if He == 512:
        assert not torch.equal(off, pbr)           # the footprints here span many texels: the mode is not a no-op


# shade_fwd_variant only moves the SH coefficients between registers and shared memory: every output keeps its bits.
# shade_group changes how many lanes share a Gaussian's samples, so the per-Gaussian sums are added in another order
# (with the mode off as well): the per-sample lights keep their bits, the sums agree to rounding.
@pytest.mark.parametrize("He", [16, 512])
def test_every_tune_variant_gives_the_same_bits(He):
    c = case(2_000, 64, He)
    lt = SoftplusLight(c["env_raw"])
    run = lambda: rendering_equation(c["base_color"], c["roughness"], c["normals"], c["viewdirs"], c["incidents"], lt,
                                     c["visibility"], c["incident_dirs"], c["incident_areas"], env_filter=True)
    with torch.no_grad():
        base = run()
        outs = [base[0], base[1]["diffuse_light"], base[1]["specular"], base[1]["global_incident_lights"]]
        for key, values in (("shade_fwd_variant", (0, 1)), ("shade_group", (8, 16, 32))):
            for v in values:
                prev = _lib.tune(key, v)
                try:
                    o = run()
                    got = [o[0], o[1]["diffuse_light"], o[1]["specular"], o[1]["global_incident_lights"]]
                finally:
                    _lib.tune(key, prev)
                if key == "shade_fwd_variant":
                    for a, b in zip(got, outs):
                        assert bits_equal(a, b), (key, v)
                else:
                    assert bits_equal(got[3], outs[3]), (key, v)
                    for a, b in zip(got[:3], outs[:3]):
                        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


# ---- 3. gradients ----------------------------------------------------------------------------------------------------------
def grads(c, kind, env_filter, views=False, cot_scale=1.0):
    leaves = {k: c[k].clone().requires_grad_(True) for k in LEAVES}
    env_raw = c["env_raw"].clone().requires_grad_(True)
    vd = (c["viewdirs_v"] if views else c["viewdirs"]).clone().requires_grad_(True)
    fn = rendering_equation_views if views else rendering_equation
    pbr, ex = fn(leaves["base_color"], leaves["roughness"], c["normals"], vd, leaves["incidents"], light(kind, c, env_raw),
                 c["visibility"], c["incident_dirs"], c["incident_areas"], env_filter=env_filter)
    pre = "vcot_" if views else "cot_"
    ((pbr * c[pre + "pbr"] * cot_scale).sum() + (ex["diffuse_light"] * c[pre + "diffuse"] * cot_scale).sum()
     + (ex["specular"] * c[pre + "specular"] * cot_scale).sum()).backward()
    out = {k: v.grad for k, v in leaves.items()}
    out.update(env_raw=env_raw.grad, viewdirs=vd.grad)
    return out


@pytest.mark.parametrize("kind", ["softplus", "fixed_rot"])
@pytest.mark.parametrize("P,N,He", [(3_000, 32, 16), (2_000, 32, 64)])
def test_backward_against_fp64_autograd(P, N, He, kind):
    c = case(P, N, He)
    got = grads(c, kind, True)
    leaves = {k: c[k].cpu().double().requires_grad_(True) for k in (*LEAVES, "viewdirs")}
    env_raw = c["env_raw"].cpu().double().requires_grad_(True)
    pbr, ex = ef.rendering_equation(leaves["base_color"], leaves["roughness"], c["normals"].cpu(), leaves["viewdirs"],
                                    leaves["incidents"], F.softplus(env_raw)[0], c["visibility"].cpu(), c["incident_dirs"].cpu(),
                                    c["incident_areas"].cpu(), transform=c["rot"].cpu() if kind == "fixed_rot" else None)
    ((pbr * c["cot_pbr"].cpu()).sum() + (ex["diffuse_light"] * c["cot_diffuse"].cpu()).sum()
     + (ex["specular"] * c["cot_specular"].cpu()).sum()).backward()
    for k in (*LEAVES, "viewdirs"):
        e = rel_l2(npy(got[k]), npy(leaves[k].grad))
        assert e < 1e-3, (k, e)
    if kind == "softplus":
        e = rel_l2(npy(got["env_raw"]), npy(env_raw.grad))
        print(f"\n[env filter bwd] He={He}: dL/denv rel {e:.2e}")
        assert e < 1e-3, e


@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


@pytest.mark.parametrize("det", [False, True])
def test_below_one_texel_the_mode_is_bitwise_off(det, request):
    if det:
        request.getfixturevalue("det_mode")
    c = case(500, 4096, 16)
    with torch.no_grad():
        for kind in ("softplus", "fixed_rot"):
            lt = light(kind, c, c["env_raw"])
            outs = [rendering_equation(c["base_color"], c["roughness"], c["normals"], c["viewdirs"], c["incidents"], lt,
                                       c["visibility"], c["incident_dirs"], c["incident_areas"], env_filter=f) for f in (False, True)]
            for k in ("diffuse_light", "specular", "global_incident_lights", "incident_lights"):
                assert bits_equal(outs[0][1][k], outs[1][1][k]), (kind, k)
            assert bits_equal(outs[0][0], outs[1][0])
    a, b = grads(c, "softplus", False), grads(c, "softplus", True)
    for k in a:
        if k == "env_raw" and not det:
            # the default mode adds dL/denv with float atomics in warp arrival order, so two calls with the mode off
            # differ in the last bits too; the deterministic mode compares bit for bit
            assert rel_l2(npy(a[k]), npy(b[k])) <= 1e-6, k
        else:
            assert bits_equal(a[k], b[k]), k


@pytest.mark.parametrize("He", [16, 64])
def test_deterministic_mode(He, det_mode):
    c = case(3_000, 32, He)
    a, b = grads(c, "softplus", True), grads(c, "softplus", True)
    for k in a:
        assert bits_equal(a[k], b[k]), k
    s = grads(c, "softplus", True, cot_scale=2.0 ** -20)
    assert torch.equal(s["env_raw"] * 2.0 ** 20, a["env_raw"])          # equivariant under power-of-two scaling
    torch.use_deterministic_algorithms(False)
    d = grads(c, "softplus", True)
    for k in a:
        assert rel_l2(npy(a[k]), npy(d[k])) <= 1e-5, k


# ---- 4. several views ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,P,N,He", [(3, 2_000, 64, 16), (9, 500, 64, 512)])
@pytest.mark.parametrize("kind", ["softplus", "fixed_rot", "per_view"])
def test_views_forward_bitwise_against_one_view_calls(V, P, N, He, kind):
    c = case(P, N, He, V=V)
    tex = F.softplus(c["env_raw"])[0]
    with torch.no_grad():
        lt = FixedLight(tex, c["rot_v"]) if kind == "per_view" else light(kind, c, c["env_raw"])
        pbr, ex = rendering_equation_views(c["base_color"], c["roughness"], c["normals"], c["viewdirs_v"], c["incidents"], lt,
                                           c["visibility"], c["incident_dirs"], c["incident_areas"], means=True, env_filter=True)
        for v in range(V):
            lv = FixedLight(tex, c["rot_v"][v]) if kind == "per_view" else lt
            one, ex1 = rendering_equation_views(c["base_color"], c["roughness"], c["normals"], c["viewdirs_v"][v:v + 1],
                                                c["incidents"], lv, c["visibility"], c["incident_dirs"], c["incident_areas"],
                                                means=True, env_filter=True)
            p1, e1 = rendering_equation(c["base_color"], c["roughness"], c["normals"], c["viewdirs_v"][v], c["incidents"], lv,
                                        c["visibility"], c["incident_dirs"], c["incident_areas"], env_filter=True)
            assert bits_equal(pbr[v], p1) and bits_equal(pbr[v], one[0])
            assert bits_equal(ex["diffuse_light"][v], e1["diffuse_light"]) and bits_equal(ex["specular"][v], e1["specular"])
            for k in shading._MEANS:
                assert bits_equal(ex[k][v], ex1[k][0]), (v, k)


@pytest.mark.parametrize("V,P,N,He", [(4, 3_000, 32, 16), (3, 1_000, 32, 64)])
def test_views_backward_equals_sum_of_one_view_calls(V, P, N, He):
    c = case(P, N, He, V=V)
    got = grads(c, "softplus", True, views=True)
    tot = {}
    for v in range(V):
        cv = dict(c, viewdirs=c["viewdirs_v"][v], cot_pbr=c["vcot_pbr"][v], cot_diffuse=c["vcot_diffuse"][v],
                  cot_specular=c["vcot_specular"][v])
        g = grads(cv, "softplus", True)
        for k in (*LEAVES, "env_raw"):
            tot[k] = tot.get(k, 0) + g[k].double()
        assert rel_l2(npy(got["viewdirs"][v]), npy(g["viewdirs"])) <= 1e-6
    for k in (*LEAVES, "env_raw"):
        assert rel_l2(npy(got[k]), npy(tot[k])) <= 1e-5, k


# ---- 5. the process default through install() ---------------------------------------------------------------------------
def test_set_env_filter_reaches_an_installed_module():
    import types
    neilf = shading.install(types.ModuleType("neilf_stand_in"))
    c = case(2_000, 64, 512)
    args = (c["base_color"], c["roughness"], c["normals"], c["viewdirs"], c["incidents"], light("fixed", c, c["env_raw"]),
            c["visibility"], c["incident_dirs"], c["incident_areas"])
    with torch.no_grad():
        off = rendering_equation(*args, env_filter=False)[0]
        on = rendering_equation(*args, env_filter=True)[0]
        prev = shading.set_env_filter(True)
        try:
            assert bits_equal(neilf.rendering_equation(*args)[0], on)
        finally:
            shading.set_env_filter(prev)
        shading.set_env_filter(False)
        assert bits_equal(neilf.rendering_equation(*args)[0], off)
        shading.set_env_filter(prev)
    assert not torch.equal(on, off)


# ---- 6. refusals ---------------------------------------------------------------------------------------------------------
def test_refusals_before_any_launch():
    lib = _lib.load()
    c = case(100, 16, 64)
    env = F.softplus(c["env_raw"])[0].contiguous()
    pyr = shading.env_pyramid(env)
    assert lib.r3dg_env_pyramid_build(None, 64, 128, pyr.data_ptr(), None) == -10001
    assert lib.r3dg_env_pyramid_build(env.data_ptr(), 0, 128, pyr.data_ptr(), None) == -10001
    assert lib.r3dg_env_pyramid_build(env.data_ptr(), 64, 128, None, None) == -10001
    a, ts, _ = shading._shade_args((c["base_color"], c["roughness"], c["normals"], c["viewdirs"], c["incidents"], env,
                                    c["visibility"], c["incident_dirs"], c["incident_areas"]), None)
    outs = [torch.empty(s, device="cuda") for s in ((100, 3), (100, 3), (100, 3), (100, 1), (100, 3), (100, 16, 3), env.shape)]
    a.dL_dpbr, a.dL_ddiffuse_light, a.dL_dspecular = outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr()
    a.dL_dbase_color, a.dL_droughness, a.dL_dviewdirs = outs[0].data_ptr(), outs[3].data_ptr(), outs[4].data_ptr()
    a.dL_dincidents, a.dL_denv = outs[5].data_ptr(), outs[6].data_ptr()
    a.env_pyramid = pyr.data_ptr()
    assert lib.r3dg_render_equation_backward(ctypes.byref(a), None) == -10001           # no pyramid workspace
    g_pyr = torch.empty_like(pyr)
    a.dL_denv_pyramid = g_pyr.data_ptr()
    small = torch.empty(lib.r3dg_shade_det_bytes(64, 128), dtype=torch.uint8, device="cuda")
    a.deterministic, a.det_work, a.det_work_bytes = 1, None, 0
    assert lib.r3dg_render_equation_backward(ctypes.byref(a), None) == -10001           # no deterministic workspace
    a.det_work, a.det_work_bytes = small.data_ptr(), small.numel()
    assert lib.r3dg_shade_filtered_det_bytes(64, 128) > small.numel()
    assert lib.r3dg_render_equation_backward(ctypes.byref(a), None) == -10001           # too small for every level
    torch.cuda.synchronize()
