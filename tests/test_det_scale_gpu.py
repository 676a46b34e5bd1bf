"""Deterministic mode at the cotangent scales training runs at.

1. Power-of-two equivariance.  The backward is linear in its cotangents, and an fp32 product with 2^-k is exact while
   nothing is subnormal, so every gradient summed in a fixed order satisfies grad(2^-k cot) == 2^-k grad(cot) bit for
   bit.  The fixed-point sums of the deterministic mode (csrc/detacc.cuh) keep that only because their unit follows
   the cotangents' scale; a fixed unit would round a training loss's faint terms (per-pixel cotangents ~2^-21) to a
   coarse grid or to zero.  The camera gradients and the shading per-Gaussian gradients never go through those sums:
   they are the controls.
2. Per-row fp64 truth of the compositor's sums (raster64.py) at unit cotangents, at a training loss's cotangents and
   at those times 2^-10, in both modes, with one bound |g - g64| <= TAU * m_row per row for all of them."""
import numpy as np
import pytest
import torch

import raster64
import test_camera_grad_gpu as cg
import test_raster_gpu as tr
import test_shading_edge_gpu as sg
import shading_edge as se
from helpers import case_inputs, edge_case, npy
from relightable3dgaussian_b200 import synth
from relightable3dgaussian_b200.rasterizer import rasterize_views

pytestmark = pytest.mark.gpu

KS = (1, 8, 21, 30)
TINY = 2.0 ** -100       # results below this (at the smaller scale) may have gone through a subnormal: not compared


@pytest.fixture
def det():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def unit_planes(t):
    """t scaled by a power of two so that max |t| lies in [1, 2) (per tensor: one plane set of one output)."""
    m = float(t.abs().max())
    return t if m == 0 else t * 2.0 ** -np.floor(np.log2(m))


def check_equivariant(tag, base, scaled, k):
    """scaled == base * 2^-k bit for bit, wherever the smaller value is above TINY (zeros must stay zeros)."""
    s = 2.0 ** -k
    for name, g in base.items():
        if g is None:
            continue
        h = scaled[name]
        want = g * s                                   # exact: a power of two
        keep = want.abs() >= TINY
        zero = g == 0
        assert torch.equal(h[zero], g[zero]), f"{tag} {name}: a zero became nonzero at k = {k}"
        bad = (h.view(torch.int32) != want.view(torch.int32)) & keep
        n = int(bad.sum())
        if n:
            d = ((h.double() - want.double()).abs() / want.double().abs().clamp_min(1e-300))[bad]
            print(f"[equivariance] {tag} {name} k={k}: {n} of {int(keep.sum())} elements differ, worst rel {float(d.max()):.3e}")
        assert n == 0, f"{tag} {name}: grad(2^-{k} cot) != 2^-{k} grad(cot) in {n} elements"


# ---- 1. equivariance -------------------------------------------------------------------------------------------------
P_EQ, W_EQ, H_EQ, S_EQ = 60_000, 320, 240, 5


def _raster_grads(V, cots, *, colors=False, cov=False, aa=False, appearance=False, surface=False, per_view=False):
    """Every gradient of one rasterize_views call with the given cotangents of its six images."""
    torch.manual_seed(0)
    leaves = cg.make_leaves(P_EQ, S_EQ, colors=colors, cov=cov, seed=3)
    if per_view:
        leaves["features"] = (leaves["features"].detach()[None] *
                              torch.linspace(0.5, 1.5, V, device="cuda")[:, None, None]).contiguous().requires_grad_(True)
    if appearance:
        for k in list(leaves):
            if k not in ("features", "shs", "colors_precomp"):
                leaves[k] = leaves[k].detach()
    cams = [synth.make_camera(v + 1, W_EQ, H_EQ, center_shift=(v % 2 == 1)) for v in range(V)]
    camt = [cg.camera_tensors(c, grad=not appearance) for c in cams]
    settings = [cg.settings_of(c, *t) for c, t in zip(cams, camt)]
    m2d = torch.zeros(V, P_EQ, 3, device="cuda", requires_grad=not appearance)
    kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
    out = rasterize_views(leaves["means3D"], m2d, leaves["opacities"], settings=settings, surface_grads=surface,
                          antialiasing=aa, **kw)
    outs = [out[i] for i in range(2, 8)]
    names = [k for k, t in leaves.items() if t.requires_grad]
    inputs = [leaves[k] for k in names]
    if not appearance:
        names += ["means2D"] + [f"{n}{v}" for v in range(V) for n in ("viewmatrix", "projmatrix", "campos")]
        inputs += [m2d] + [t for ts in camt for t in ts]
    gs = torch.autograd.grad(outs, inputs, grad_outputs=cots, allow_unused=True)
    return dict(zip(names, gs))


def _base_cots(V, surface):
    g = torch.Generator().manual_seed(11)
    shapes = [(V, 3, H_EQ, W_EQ), (V, 1, H_EQ, W_EQ), (V, 1, H_EQ, W_EQ), (V, S_EQ, H_EQ, W_EQ), (V, 3, H_EQ, W_EQ),
              (V, 3, H_EQ, W_EQ)]
    cots = [unit_planes(torch.randn(s, generator=g)).cuda() for s in shapes]
    if not surface:
        cots[4].zero_(); cots[5].zero_()
    return cots


RASTER_CALLS = {
    "one-view-sh": dict(V=1),
    "views3-per-view-features": dict(V=3, per_view=True),
    "precomp": dict(V=1, colors=True, cov=True),
    "antialiasing": dict(V=1, aa=True),
    "appearance-only": dict(V=1, appearance=True),
    "appearance-only-views3": dict(V=3, appearance=True),
    "surface": dict(V=1, surface=True),
}


@pytest.mark.parametrize("call", list(RASTER_CALLS))
def test_raster_backward_power_of_two_equivariant(det, call):
    kw = dict(RASTER_CALLS[call])
    V = kw.pop("V")
    cots = _base_cots(V, kw.get("surface", False))
    base = _raster_grads(V, cots, **kw)
    assert any(float(g.abs().max()) > 0 for g in base.values() if g is not None)
    for k in KS:
        check_equivariant(call, base, _raster_grads(V, [c * 2.0 ** -k for c in cots], **kw), k)


@pytest.mark.parametrize("name", ["seam_poles", "seam_poles_64"])
def test_shading_backward_power_of_two_equivariant(det, name):
    """DirectLightMap 16x32 (dL/denv in shared-memory accumulators) and 64x128 (global accumulators)."""
    t = se.inputs(sg.CASES[name], "cuda")
    for c in se.COTS:
        t["cot_" + c] = unit_planes(t["cot_" + c])
    grads = lambda rec: {k: v for k, v in rec.items() if k.startswith("grad_")}         # noqa: E731
    base = grads(sg.run_ours(t))
    assert float(base["grad_tex"].abs().max()) > 0
    for k in KS:
        ts = dict(t, **{"cot_" + c: t["cot_" + c] * 2.0 ** -k for c in se.COTS})
        check_equivariant(name, base, grads(sg.run_ours(ts)), k)


# ---- 2. per-row fp64 truth ---------------------------------------------------------------------------------------------
# One bound for every cotangent set and both modes, from the worst row measured on an H100 SXM (80 GB, 700 W) in the
# default mode at unit cotangents over the scenes below: TAU_MEASURED (the worst |g - g64| / m_row).  TAU leaves 4x.
TAU_MEASURED = 5.2e-5    # shell-20k-160x120-S5, dL_dopacity (the other scenes: opaque-S5 5.3e-6, inside-x1 1.2e-5)
TAU = 4 * TAU_MEASURED
OUTPUTS = ("dL_dcolors", "dL_dfeatures", "dL_dopacity", "dL_dmeans2D", "dL_dcov3D")


def _precomp(kw):
    """colors_precomp + cov3D_precomp in place of SH and scales / rotations (the scene's own covariance)."""
    kw = dict(kw)
    if "shs" in kw:
        P = kw["means3D"].shape[0]
        kw["colors_precomp"] = torch.rand(P, 3, generator=torch.Generator().manual_seed(7)).numpy()
        del kw["shs"]
    if "scales" in kw:
        C = raster64.aa_oracle.cov3d_of(torch.as_tensor(kw.pop("scales")).double(),
                                        torch.as_tensor(kw.pop("rotations")).double(), kw.get("scale_modifier", 1.0))
        kw["cov3D_precomp"] = torch.stack([C[:, 0, 0], C[:, 0, 1], C[:, 0, 2], C[:, 1, 1], C[:, 1, 2], C[:, 2, 2]],
                                          1).float().numpy()
    kw["scale_modifier"] = 1.0
    return kw


def _shell_20k():
    sc, cam = case_inputs(20_000, 160, 120, 5, view=1)
    kw = dict(means3D=npy(sc.means3D), opacities=npy(sc.opacities), viewmatrix=npy(cam.viewmatrix),
              projmatrix=npy(cam.projmatrix), campos=npy(cam.campos), bg=np.array([0.0, 0.5, 1.0], np.float32),
              W=160, H=120, tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy, shs=npy(sc.shs),
              scales=npy(sc.scales), rotations=npy(sc.rotations), features=npy(sc.features))
    return kw


SCENES = {"opaque-S5": lambda: edge_case("opaque-S5")[0], "inside-x1": lambda: edge_case("inside-x1")[0],
          "thresholds": lambda: edge_case("thresholds")[0], "shell-20k-160x120-S5": _shell_20k}


def _training_cots(o, S, W, H):
    """Cotangents of L1(color, gt) + 0.2 (1 - ssim(color, gt)) + L1 on three feature channels (or all S < 3) at the
    kernel's own images."""
    from relightable3dgaussian_b200 import losses
    g = torch.Generator(device="cuda").manual_seed(5)
    gt = torch.rand(3, H, W, device="cuda", generator=g)
    gf = torch.rand(min(3, S), H, W, device="cuda", generator=g)
    col = o["color"].detach().clone().requires_grad_(True)
    feat = o["feature"].detach().clone().requires_grad_(True)
    loss = (col - gt).abs().mean() + 0.2 * (1.0 - losses.ssim(col, gt)) + (feat[:min(3, S)] - gf).abs().mean()
    dc, df = torch.autograd.grad(loss, [col, feat])
    z = torch.zeros(1, H, W, device="cuda")
    return [dc, z, z.clone(), df]


@pytest.mark.parametrize("scene", list(SCENES))
def test_compositor_rows_match_fp64_truth(scene):
    from relightable3dgaussian_b200 import _C_raster as C
    kw = _precomp(SCENES[scene]())
    W, H = kw["W"], kw["H"]
    S = kw["features"].shape[1] if kw.get("features") is not None else 0
    assert S >= 1
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        o = tr.run_ours(C, **kw)
        P = kw["means3D"].shape[0]
        mid = lambda n: o["mid"](n)                                                      # noqa: E731
        st = dict(point_list=mid("point_list"), ranges=mid("ranges"), n_contrib=mid("n_contrib"),
                  means2D=mid("means2D"), conic_opacity=mid("conic_opacity"), rgb=mid("rgb"), depths=mid("depths"),
                  features=torch.as_tensor(kw["features"]).cuda())
        bg = torch.as_tensor(kw["bg"]).cuda()
        walks = raster64.walks_of(st, W, H)
        # the oracle first: n_contrib and the images on every pixel that is not ambiguous
        amb = torch.zeros(H * W, dtype=torch.bool, device="cuda")
        img = torch.cat([o["color"], o["opacity"], o["depth"], o["feature"]], 0).reshape(5 + S, -1)
        rows = torch.zeros(P, dtype=torch.bool, device="cuda")
        for wk in walks:
            amb[wk.pix] = wk.ambiguous
            ok = ~wk.ambiguous
            assert bool(wk.nc_ok[ok].all()), f"{scene}: fp64 disagrees with n_contrib on a pixel that is not ambiguous"
            ours = wk.composite(st, bg, S, wk.alpha)
            err = (ours - img[:, wk.pix].T.double()).abs()[ok]
            assert err.numel() == 0 or float(err.max()) <= 1e-5, (scene, float(err.max()))
            rows[wk.ids[wk.valid & ok[:, None]]] = True
        crit = {k: sum(int(wk.criteria[k].sum()) for wk in walks) for k in walks[0].criteria}
        frac = float(amb.sum()) / (H * W)
        print(f"[fp64] {scene}: {int(rows.sum())} rows composited by unambiguous pixels, {int(amb.sum())} ambiguous "
              f"pixels {crit} ({100 * frac:.3f} %), given zero cotangents")
        live = (~amb).float().view(1, H, W)
        keep = rows
        view = torch.as_tensor(kw["viewmatrix"]).cuda()
        jac = raster64.cov3d_jacobian(torch.as_tensor(kw["means3D"]).cuda(), torch.as_tensor(kw["cov3D_precomp"]).cuda(),
                                      view, W, H, kw["tan_fovx"], kw["tan_fovy"])
        gu = torch.Generator().manual_seed(2)
        unit = [torch.randn(c, H, W, generator=gu).cuda() for c in (3, 1, 1, S)]
        train = _training_cots(o, S, W, H)
        sets = {"unit": unit, "training": train, "training*2^-10": [c * 2.0 ** -10 for c in train]}
        sets = {k: [c * live for c in cs] for k, cs in sets.items()}
        failures = {}
        for sname, cots in sets.items():
            truth = raster64.row_truth(st, walks, cots, bg, W, H, S, jac)
            for mode in (False, True):
                torch.use_deterministic_algorithms(mode)
                g = tr.run_ours(C, cots=cots, **kw)["grads"]
                worst, nfail = 0.0, 0
                for name in OUTPUTS:
                    g64, m = truth[name]
                    ours = g[name].reshape(P, -1)[:, :g64.shape[1]].double()
                    r = ((ours - g64).abs() / m.clamp_min(1e-300))[keep]
                    r = torch.where((m[keep] == 0) & (ours[keep] == 0), torch.zeros_like(r), r)
                    bad = (r > TAU).any(1)
                    nfail += int(bad.sum())
                    w = float(r.max()) if r.numel() else 0.0
                    worst = max(worst, w)
                    if bad.any():
                        print(f"[fp64] {scene} {'det' if mode else 'default'} {sname} {name}: {int(bad.sum())} rows "
                              f"over tau, worst ratio {w:.3e}")
                print(f"[fp64] {scene} {'det' if mode else 'default'} {sname}: {nfail} row-outputs over tau = {TAU:.1e} "
                      f"of {int(keep.sum())} rows, worst |g - g64| / m_row {worst:.3e}")
                failures[(mode, sname)] = nfail
    finally:
        torch.use_deterministic_algorithms(prev)
    assert frac < 0.01, f"{scene}: {100 * frac:.3f} % of the pixels are ambiguous"
    assert not any(failures.values()), failures
