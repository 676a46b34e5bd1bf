"""The antialiased rasterizer mode (`antialiasing=True`) on the GPU, through an exact decomposition.

Run A is the mode on with opacities o.  Run B is the mode off with the opacities o' that A stored in its record
(debug_intermediate("conic_opacity")[:, 3] = o rho).  Every compositor reads only that record, so in deterministic
mode:
  * every forward output of B equals A's bit for bit, and A's geometry (conic, radii, tile lists) is that of the mode
    off with o; A's stored opacity is o rho of the fp64 closed form (tests/aa_oracle.py);
  * the gradients that do not go through rho (means2D, SH, features, colours, projmatrix, campos) equal B's bit for
    bit; dL/do = rho dL/do'; and the gradients of means3D, scales, rotations, cov3D_precomp and the view matrix are B's
    plus the fp64 autograd of rho weighted by o dL/do'.
The file also checks several views, frozen geometry, surface gradients, the deferred-count repair, reproducibility
and the default (float-atomic) mode."""
import warnings

import numpy as np
import pytest
import torch

import aa_oracle
from helpers import EDGE_CASES, edge_case
from relightable3dgaussian_b200 import _C_raster, synth
from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer, set_deferred_count

pytestmark = pytest.mark.gpu

GRADS = ("means2D", "colors_precomp", "opacities", "means3D", "features", "cov3D_precomp", "shs", "scales", "rotations",
         "viewmatrix", "projmatrix", "campos")
OUT = ("color", "opacity", "depth", "feature", "normal", "surface_xyz", "weights", "radii")
EPS = 2.0 ** -24
# Bounds measured on an H100 over every scene below (see each use).
RHO_TOL = 64 * EPS          # stored o rho against o rho_64, relative, times (1 + conditioning of det0)
# rel-L2 of the geometry gradients against B's plus the fp64 rho term, per-Gaussian gradients over the well-conditioned
# rows (see well_conditioned).  The view matrix, a sum over all rows, is compared relative to |B's| + |the rho term|:
# the two nearly cancel on some scenes.  The H100 showed up to 9.9e-5 (`needles`, means3D) and 2.8e-4 (`strip-9x4`,
# view matrix in plain rel-L2) in deterministic mode.
CHAIN_TOL = 5e-4
# The same in the default mode, where A and B are two runs whose float-atomic sums differ: 1.04e-3 (`needles`, means3D)
DEFAULT_TOL = 2e-3


@pytest.fixture
def det_mode():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def bits_equal(a, b):
    if a is None or b is None:
        return a is None and b is None
    a, b = a.contiguous(), b.contiguous()
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return a.shape == b.shape and torch.equal(a, b)


def rel_l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def to_cuda(kw):
    d = {k: (torch.from_numpy(np.ascontiguousarray(v)).float().cuda() if isinstance(v, np.ndarray) else v)
         for k, v in kw.items()}
    if d["opacities"].dim() == 1:
        d["opacities"] = d["opacities"][:, None].contiguous()
    return d


def far_scene(precomp):
    """Sub-pixel Gaussians: the shell seen from 5x further away than usual (median rho ~ 0.14)."""
    sc = synth.make_scene(20_000, "shell-v1", 7, 5)
    cam = synth.make_camera(1, 320, 240, radius=20.0)
    d = dict(means3D=sc.means3D, opacities=sc.opacities, viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix,
             campos=cam.campos, bg=torch.tensor([0.1, 0.4, 0.7]), W=cam.image_width, H=cam.image_height,
             tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy, features=sc.features, scale_modifier=1.0)
    if precomp:
        sig = aa_oracle.cov3d_of(sc.scales.double(), sc.rotations.double())
        d["cov3D_precomp"] = sig[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].float()
        d["colors_precomp"] = torch.rand(sc.means3D.shape[0], 3, generator=torch.Generator().manual_seed(1))
    else:
        d.update(shs=sc.shs, scales=sc.scales, rotations=sc.rotations)
    g = torch.Generator().manual_seed(2)
    cots = [torch.randn(c, cam.image_height, cam.image_width, generator=g) for c in (3, 1, 1, 5)]
    return {k: (v.float().contiguous().cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}, \
        [c.cuda() for c in cots]


def scene(name):
    if name.startswith("far-"):
        d, cots = far_scene(name == "far-precomp")
    else:
        kw, cots = edge_case(name)
        d, cots = to_cuda(kw), [torch.from_numpy(c).float().cuda() for c in cots]
    if d["opacities"].dim() == 1:
        d["opacities"] = d["opacities"][:, None].contiguous()
    if d.get("features") is None:
        d["features"] = torch.empty(d["means3D"].shape[0], 0, device="cuda")
    return d, cots


def run(d, opac, aa, cots, backward=True, surface=None, **bkw):
    """Forward (and backward with camera gradients) through the C ABI's host layer.  `surface` = (g_normal, g_xyz)
    differentiates the pseudo-normal and surface-xyz outputs too."""
    E = torch.empty(0, device="cuda")
    g = lambda k: d.get(k, E)
    P, S = d["means3D"].shape[0], d["features"].shape[1]
    o = _C_raster.rasterize_gaussians(d["bg"], d["means3D"], d["features"], g("colors_precomp"), opac, g("scales"),
                                      g("rotations"), d["scale_modifier"], g("cov3D_precomp"), d["viewmatrix"],
                                      d["projmatrix"], d["tan_fovx"], d["tan_fovy"], d["cx"], d["cy"], d["H"], d["W"],
                                      g("shs"), 3, d["campos"], False, True, False, antialiasing=aa)
    r = dict(zip(("num_rendered", "n_contrib", "color", "opacity", "depth", "feature", "normal", "surface_xyz",
                  "weights", "radii"), o[:10]))
    mid = lambda n: _C_raster.debug_intermediate(n, P, S, d["W"], d["H"], o[10], o[12], o[11], o[0])
    r.update(conic=mid("conic_opacity"), point_list=mid("point_list"), ranges=mid("ranges"))
    if backward:
        kw = dict(bkw)
        if kw.get("geometry", True):
            kw["cam_grads"] = True
            if surface is not None:
                kw["surface"] = (surface[0], surface[1], o[3], o[4], d["cx"], d["cy"])
        gr = _C_raster.rasterize_gaussians_backward(d["bg"], d["means3D"], d["features"], o[9], g("colors_precomp"),
                                                    g("scales"), g("rotations"), d["scale_modifier"],
                                                    g("cov3D_precomp"), d["viewmatrix"], d["projmatrix"], d["tan_fovx"],
                                                    d["tan_fovy"], *cots, g("shs"), 3, d["campos"], o[10], o[0], o[11],
                                                    o[12], True, False, antialiasing=aa, **kw)
        r["grads"] = dict(zip(GRADS, gr))
    torch.cuda.synchronize()
    return r


def rho64(d, inputs=None):
    """rho of the fp64 closed form, differentiable in the fp64 copies `inputs` (made here when not given)."""
    if inputs is None:
        inputs = {k: d[k].double().detach().requires_grad_(True)
                  for k in ("means3D", "viewmatrix", "scales", "rotations", "cov3D_precomp") if k in d}
    rho = aa_oracle.rho(inputs["means3D"], inputs["viewmatrix"], d["W"], d["H"], d["tan_fovx"], d["tan_fovy"],
                        scales=inputs.get("scales"), rotations=inputs.get("rotations"),
                        cov3D=inputs.get("cov3D_precomp"), scale_modifier=d["scale_modifier"])
    return rho, inputs


def conditioning(d):
    """(|a0| + |c0|)^2 / det0 of every Gaussian in fp64: how much the fp32 rounding of the 2D covariance can move r;
    infinite where the 2D covariance before the dilation is not positive definite."""
    with torch.no_grad():
        x = {k: d[k].double() for k in ("means3D", "viewmatrix", "scales", "rotations", "cov3D_precomp") if k in d}
        sig = (aa_oracle.cov3d_from_six(x["cov3D_precomp"]) if "cov3D_precomp" in x
               else aa_oracle.cov3d_of(x["scales"], x["rotations"], d["scale_modifier"]))
        a0, b, c0 = aa_oracle.cov2d(x["means3D"], sig, x["viewmatrix"], d["W"], d["H"], d["tan_fovx"], d["tan_fovy"])
        kappa = (a0.abs() + c0.abs()) ** 2 / (a0 * c0 - b * b).clamp_min(1e-300)
        return torch.where((a0 > 0) & (c0 > 0), kappa, torch.full_like(kappa, float("inf")))


def well_conditioned(kappa, rho):
    """Rows whose fp32 rho the fp64 closed form predicts to first order: det0 conditioned to <= 1e4 and rho not
    within 5 % of the floor, where the fp32 and fp64 floor decisions may differ and switch rho's gradient on or off."""
    return (kappa <= 1e4) & ((rho / aa_oracle.FLOOR ** 0.5 - 1).abs() > 0.05)


def decomposition(d, cots, det, surface=None):
    """Runs A, B and the mode off with o; checks the decomposition.  Returns A (for further checks)."""
    o = d["opacities"]
    A = run(d, o, True, cots, surface=surface)
    vis = A["radii"] > 0
    o2 = torch.where(vis[:, None], A["conic"][:, 3:4], o).contiguous()
    B = run(d, o2, False, cots, surface=surface)
    C = run(d, o, False, cots, backward=False)
    # ---- forward
    assert A["num_rendered"] == B["num_rendered"] == C["num_rendered"]
    for k in OUT + ("n_contrib",):
        if det or k in ("radii", "n_contrib", "color", "opacity", "depth", "feature", "normal", "surface_xyz"):
            assert bits_equal(A[k], B[k]), k
        else:
            torch.testing.assert_close(A[k], B[k], rtol=1e-3, atol=1e-6)
    assert bits_equal(A["conic"][:, :3], C["conic"][:, :3])
    for k in ("radii", "point_list", "ranges"):
        assert bits_equal(A[k], C[k]), k
    rho, inputs = rho64(d)
    want = (o[:, 0].double() * rho).detach()
    on = vis & (rho > aa_oracle.FLOOR ** 0.5 * (1 + 1e-3)) & (want > 0)
    kappa = conditioning(d)
    err = (A["conic"][:, 3].double() - want).abs() / want.clamp_min(1e-300)
    fin = on & torch.isfinite(kappa)
    assert bool((err[fin] <= RHO_TOL * (1 + kappa[fin])).all()), float((err[fin] / (1 + kappa[fin])).max() / EPS)
    # ---- gradients
    gA, gB = A["grads"], B["grads"]
    same = ["means2D", "features", "shs", "colors_precomp", "projmatrix", "campos"]
    for k in same:
        if gA[k] is not None and gA[k].numel():
            assert (bits_equal(gA[k], gB[k]) if det else rel_l2(gA[k], gB[k]) <= 1e-3), k
    # dL/do = rho dL/do' (rho of the backward's own fp32 covariance: the same conditioning bound as the forward)
    want_do = rho.detach() * gB["opacities"][:, 0].double()
    e_do = (gA["opacities"][:, 0].double() - want_do).abs()
    big = on & torch.isfinite(kappa) & (want_do.abs() > 0)
    if det:
        assert bool((e_do[big] <= RHO_TOL * (1 + kappa[big]) * want_do[big].abs()).all()), \
            float((e_do[big] / want_do[big].abs() / (1 + kappa[big])).max() / EPS)
    else:
        assert rel_l2(gA["opacities"][:, 0], want_do) <= 1e-3
    # geometry: B's gradients plus the fp64 autograd of rho weighted by o dL/do'
    w = o[:, 0].double() * gB["opacities"][:, 0].double()
    names = list(inputs)
    extra = dict(zip(names, torch.autograd.grad((w * rho).sum(), [inputs[k] for k in names], allow_unused=True)))
    well = well_conditioned(kappa, rho.detach())
    for k in names:
        got, base = gA[k], gB[k]
        if k == "viewmatrix":
            got, base = got.view(4, 4), base.view(4, 4)
        term = extra[k] if extra[k] is not None else torch.zeros_like(base, dtype=torch.float64)
        if k == "scales":           # dL_dscales is the gradient of the modified scale (the reference's convention)
            term = term / d["scale_modifier"]
        ref = base.double() + term
        if k == "viewmatrix" and not det and bool((kappa[vis] > 1e4).any()):
            # rows whose fp32 det0 is rounding noise (`needles`) have a huge, noise-driven rho term; summed into the view
            # matrix it follows the float-atomic order of dL/d(o rho), which differs between A and B (measured 7 %)
            continue
        if k == "viewmatrix":
            e = ((got.double() - ref).norm() / (base.double().norm() + term.norm()).clamp_min(1e-30)).item()
        else:
            e = rel_l2(got[well], ref[well])
        assert e <= (CHAIN_TOL if det else DEFAULT_TOL), (k, e)
    for t in list(gA.values()) + [A[k] for k in OUT]:
        if t is not None and t.is_floating_point():
            assert bool(torch.isfinite(t).all())
    return A


SCENES = list(EDGE_CASES) + ["far-sr", "far-precomp"]


@pytest.mark.parametrize("name", SCENES)
def test_decomposition_deterministic(name, det_mode):
    d, cots = scene(name)
    decomposition(d, cots, det=True)


@pytest.mark.parametrize("name", ["far-sr", "far-precomp", "needles", "precomp", "inside-x1"])
def test_decomposition_default_mode(name):
    d, cots = scene(name)
    decomposition(d, cots, det=False)


@pytest.mark.parametrize("name", ["far-sr", "far-precomp"])
def test_reproducible_and_finite(name, det_mode):
    d, cots = scene(name)
    a = run(d, d["opacities"], True, cots)
    b = run(d, d["opacities"], True, cots)
    for k in OUT + ("n_contrib", "conic"):
        assert bits_equal(a[k], b[k]), k
    for k, t in a["grads"].items():
        assert bits_equal(t, b["grads"][k]), k
        if t is not None:
            assert bool(torch.isfinite(t).all()), k
    assert float(a["conic"][a["radii"] > 0, 3].div(d["opacities"][a["radii"] > 0, 0]).median()) < 0.5   # rho << 1


def test_surface_grads_decomposition(det_mode):
    d, cots = scene("far-sr")
    g = torch.Generator().manual_seed(11)
    surface = tuple(torch.randn(3, d["H"], d["W"], generator=g).cuda() * s for s in (1.0, 0.1))
    decomposition(d, cots, det=True, surface=surface)


def test_frozen_geometry_gives_the_full_backwards_appearance_gradients(det_mode):
    for name in ("far-sr", "far-precomp"):
        d, cots = scene(name)
        full = run(d, d["opacities"], True, cots)["grads"]
        app = run(d, d["opacities"], True, cots, geometry=False)["grads"]
        for k in ("features", "colors_precomp", "shs"):
            if app[k] is not None:
                assert bits_equal(app[k], full[k]), (name, k)


def test_three_views_equal_three_one_view_calls(det_mode):
    sc = synth.make_scene(30_000, "shell-v1", 3, 5)
    W, H = 320, 240
    cams = [synth.make_camera(k, W, H, radius=12.0 + 8 * k) for k in range(3)]
    leaf = lambda t: t.float().contiguous().cuda()
    base = dict(means3D=leaf(sc.means3D), opacities=leaf(sc.opacities), shs=leaf(sc.shs), scales=leaf(sc.scales),
                rotations=leaf(sc.rotations), features=leaf(sc.features), scale_modifier=1.0, W=W, H=H)
    g = torch.Generator().manual_seed(4)
    cots = [[torch.randn(c, H, W, generator=g).cuda() for c in (3, 1, 1, 5)] for _ in cams]
    bgs = [torch.tensor([0.1 * k, 0.4, 0.7], device="cuda") for k in range(3)]
    per = []
    for k, cam in enumerate(cams):
        d = dict(base, viewmatrix=leaf(cam.viewmatrix), projmatrix=leaf(cam.projmatrix), campos=leaf(cam.campos),
                 bg=bgs[k], tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy)
        per.append(run(d, base["opacities"], True, cots[k]))
    E = torch.empty(0, device="cuda")
    table = [(c.tanfovx, c.tanfovy, c.cx, c.cy) for c in cams]
    vm, pm, cp = (torch.stack([leaf(getattr(c, n)) for c in cams]) for n in ("viewmatrix", "projmatrix", "campos"))
    bg = torch.stack(bgs)
    o = _C_raster.rasterize_views(bg, base["means3D"], base["features"], E, base["opacities"], base["scales"],
                                  base["rotations"], 1.0, E, vm, pm, table, H, W, base["shs"], 3, cp, False, True,
                                  antialiasing=True)
    for v in range(3):
        for i, k in enumerate(("color", "opacity", "depth", "feature", "normal", "surface_xyz", "weights", "radii"), 2):
            assert bits_equal(o[i][v], per[v][k]), (k, v)
    stack = lambda j: torch.stack([c[j] for c in cots])
    gr = _C_raster.rasterize_views_backward(bg, base["means3D"], base["features"], E, base["scales"], base["rotations"],
                                            1.0, E, vm, pm, table, stack(0), stack(1), stack(2), stack(3), base["shs"],
                                            3, cp, o[10], o[11], o[12], True, cam_grads=True, antialiasing=True)
    got = dict(zip(GRADS, gr))
    for v in range(3):
        assert bits_equal(got["means2D"][v], per[v]["grads"]["means2D"]), v
        for k in ("viewmatrix", "projmatrix", "campos"):
            assert bits_equal(got[k][v].reshape(-1), per[v]["grads"][k].reshape(-1)), (k, v)
    for k in ("opacities", "means3D", "features", "scales", "rotations"):
        ref = per[0]["grads"][k].clone()
        for v in (1, 2):
            ref += per[v]["grads"][k]
        assert bits_equal(got[k], ref), k
    ref = per[0]["grads"]["shs"] + per[1]["grads"]["shs"] + per[2]["grads"]["shs"]
    assert rel_l2(got["shs"], ref) <= 1e-6           # rebuilt from the views' rank-1 factors


def test_deferred_overflow_repair_reruns_with_the_mode_on(det_mode):
    """Learn the instance counts on small Gaussians, then boost the scales 20x so that the deferred forward overflows
    its binning buffer: the backward re-runs the forward, in the antialiased mode, and gives the synchronous call's
    gradients."""
    P, W, H, S = 3000, 160, 120, 5
    sc = synth.make_scene(P, seed=2, S=S)
    base = {k: getattr(sc, k).cuda().contiguous().requires_grad_(True)
            for k in ("means3D", "opacities", "shs", "scales", "rotations", "features")}
    big = dict(base, scales=(base["scales"].detach() * 20.0).requires_grad_(True))
    g = torch.Generator().manual_seed(9)
    cot = [torch.randn(c, H, W, generator=g).cuda() for c in (3, 1, 1, S)]

    def one_view(leaves, cam):
        vm, pm, cp = (t.cuda().contiguous() for t in (cam.viewmatrix, cam.projmatrix, cam.campos))
        rs = GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                           torch.tensor([0.1, 0.4, 0.7], device="cuda"), 1.0, vm, pm, 3, cp, False,
                                           True, True, False)
        m2d = torch.zeros(P, 3, device="cuda", requires_grad=True)
        kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
        out = GaussianRasterizer(rs, antialiasing=True)(leaves["means3D"], m2d, leaves["opacities"], **kw)
        loss = sum((out[i] * c).sum() for i, c in zip((2, 3, 4, 5), cot))
        return dict(zip(list(leaves) + ["means2D"], torch.autograd.grad(loss, list(leaves.values()) + [m2d])))

    cam = synth.make_camera(2, W, H)
    _C_raster._state.clear()
    want = one_view(big, cam)
    _C_raster._state.clear()
    set_deferred_count(True)
    old = _C_raster._HEADROOM
    try:
        _C_raster._HEADROOM = 1.0
        for i in range(_C_raster._LEARN + 1):
            one_view(base, synth.make_camera(i % 8, W, H))
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            got = one_view(big, cam)
        assert any("re-run" in str(x.message) for x in w), [str(x.message) for x in w]
        for k, t in want.items():
            e = rel_l2(got[k], t)
            assert e <= 1e-6, (k, e)
    finally:
        _C_raster._HEADROOM = old
        set_deferred_count(False)
        _C_raster._state.clear()
