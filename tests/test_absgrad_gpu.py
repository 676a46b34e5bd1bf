"""Absolute screen-space gradients (absgrad) on the GPU.

Off is off and on changes nothing else; the sums against the fp64 truth of absgrad64.py (per row, relative to the
row's sum of term magnitudes, see TAU) on every edge-case scene and a dense shell scene, at unit and training-scale cotangents, in both modes,
also antialiased and with the surface cotangents; rows not composited are +0; three views equal three one-view calls;
deterministic mode is reproducible and power-of-two equivariant; the attribute accumulates over backward calls and
survives the deferred-count repair; the densification statistic uses it."""
import warnings

import numpy as np
import pytest
import torch

import absgrad64
import raster64
import surface_oracle
import test_camera_grad_gpu as cg
from helpers import EDGE_CASES, case_inputs, edge_case, npy
from relightable3dgaussian_b200 import _C_raster, _lib, densify, synth
from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_views,
                                                   set_deferred_count)

pytestmark = pytest.mark.gpu

# |absgrad - fp64| <= TAU * m_row per row and component, m_row the row's sum of the magnitudes of the products each
# dL/dmean2D term is made of (raster64.row_truth's yardstick of the signed sums, >= fp64 absgrad): each |term| is off by
# at most what the signed term is.  Relative to the fp64 absgrad itself the error reached ~1e-3 (needles, strip-7x5): a
# term formed with cancellation (dL/dalpha = (D - A) T - ...) is small next to its products, and its fp32 error is
# relative to those.  Measured on an H100 80GB HBM3 at 700 W over every scene and variant below: up to 7.9e-4 in
# deterministic mode (strip-7x5) and 1.8e-3 in the default mode (strip-1x37 with surface cotangents); the bounds are
# about 2.5 times those.  Antialiased, the needle-like rows of the strip scenes (whose rho is dominated by rounding, see
# tests/test_antialiasing_gpu.py) reached 5.6e-3 (strip-9x4, training cotangents): TAU_AA.
TAU = {True: 2e-3, False: 4e-3}
TAU_AA = 1.5e-2
P0, W0, H0 = 40_000, 320, 240


@pytest.fixture
def det():
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(prev)


def _grads(leaves, cam, cot, V=1, det_mode=False, retain=False, twice=False, **kw):
    """Every gradient of one GaussianRasterizer call (V = 1) or one rasterize_views call over V cameras, and the means2D
    tensor (whose .absgrad the backward may have set)."""
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det_mode)
    try:
        P = leaves["means3D"].shape[0]
        other = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
        if V == 1:
            vm, pm, cp = cg.camera_tensors(cam, grad=True)
            m2d = torch.zeros(P, 3, device="cuda", requires_grad=True)
            out = GaussianRasterizer(cg.settings_of(cam, vm, pm, cp), **kw)(leaves["means3D"], m2d, leaves["opacities"],
                                                                           **other)
            cams = [vm, pm, cp]
        else:
            camt = [cg.camera_tensors(c, grad=False) for c in cam]
            m2d = torch.zeros(V, P, 3, device="cuda", requires_grad=True)
            out = rasterize_views(leaves["means3D"], m2d, leaves["opacities"],
                                  settings=[cg.settings_of(c, *t) for c, t in zip(cam, camt)], **other, **kw)
            cams = []
        loss = sum((out[i] * c).sum() for i, c in zip((2, 3, 4, 5), cot))
        inputs = list(leaves.values()) + [m2d] + cams
        g = torch.autograd.grad(loss, inputs, retain_graph=retain or twice)
        if twice:
            torch.autograd.grad(loss, inputs)
        torch.cuda.synchronize()
        names = list(leaves) + ["means2D"] + (["viewmatrix", "projmatrix", "campos"] if cams else [])
        return dict(zip(names, g)), m2d, out
    finally:
        torch.use_deterministic_algorithms(prev)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("S", [5, 14])
def test_off_is_off_and_on_changes_nothing_else(S):
    """S = 14 covers the deterministic absgrad compositor that runs 3 CTAs per SM instead of 4."""
    leaves = cg.make_leaves(P0, S, seed=3)
    cam = synth.make_camera(1, W0, H0)
    cot = cg.cotangents(H0, W0, S)
    for det_mode in (True, False):
        base, m_base, out_base = _grads(leaves, cam, cot, det_mode=det_mode)
        off, m_off, out_off = _grads(leaves, cam, cot, det_mode=det_mode, absgrad=False)
        on, m_on, out_on = _grads(leaves, cam, cot, det_mode=det_mode, absgrad=True)
        assert not hasattr(m_base, "absgrad") and not hasattr(m_off, "absgrad")
        assert m_on.absgrad.shape == (P0, 2) and bool((m_on.absgrad >= 0).all())
        for i in range(2, 9 if det_mode else 8):          # (default mode: out_weights sums with float atomics)
            assert _bits_equal(out_off[i], out_base[i]) and _bits_equal(out_on[i], out_base[i]), i
        for k, t in base.items():
            for name, g in (("off", off[k]), ("on", on[k])):
                if det_mode:
                    assert _bits_equal(g, t), (k, name)
                else:      # float atomics: two runs differ in summation order only
                    e = float((g - t).norm() / t.norm().clamp_min(1e-30))
                    assert e <= 1e-5, (k, name, e)
        # absgrad bounds the signed sum componentwise (up to fp32 rounding of the two sums)
        g = on["means2D"][:, :2].abs()
        assert bool((m_on.absgrad >= g * (1 - 1e-4) - 1e-30).all())


def _training_cots(o, S, W, H):
    """Cotangents of L1(color, gt) + 0.2 (1 - ssim(color, gt)) + L1 of the features at the kernel's own images."""
    from relightable3dgaussian_b200 import losses
    g = torch.Generator(device="cuda").manual_seed(5)
    gt = torch.rand(3, H, W, device="cuda", generator=g)
    col = o["color"].detach().clone().requires_grad_(True)
    loss = (col - gt).abs().mean() + 0.2 * (1.0 - losses.ssim(col, gt))
    dc, = torch.autograd.grad(loss, [col])
    df = torch.sign(o["feature"].detach() - 0.5) / max(1, o["feature"].numel())
    z = torch.zeros(1, H, W, device="cuda")
    return [dc, z, z.clone(), df]


def _shell():
    sc, cam = case_inputs(20_000, 160, 120, 5, view=1)
    kw = dict(means3D=npy(sc.means3D), opacities=npy(sc.opacities), viewmatrix=npy(cam.viewmatrix),
              projmatrix=npy(cam.projmatrix), campos=npy(cam.campos), bg=np.array([0.0, 0.5, 1.0], np.float32),
              W=160, H=120, tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy, shs=npy(sc.shs),
              scales=npy(sc.scales), rotations=npy(sc.rotations), features=npy(sc.features))
    return kw


SCENES = {**{n: (lambda n=n: edge_case(n)[0]) for n in EDGE_CASES}, "shell-20k-160x120-S5": _shell}


def _run(kw, cots=None, aa=False, surface=None):
    """Forward, and with `cots` the backward with absgrad, through _C_raster: the outputs, the intermediates and
    (grads, absgrad)."""
    C = _C_raster
    dev = lambda x: None if x is None else torch.as_tensor(x).cuda().contiguous()       # noqa: E731
    P = kw["means3D"].shape[0]
    feats = dev(kw.get("features")) if kw.get("features") is not None else torch.empty((P, 0), device="cuda")
    a = [dev(kw["bg"]), dev(kw["means3D"]), feats, dev(kw.get("colors_precomp")), dev(kw["opacities"]),
         dev(kw.get("scales")), dev(kw.get("rotations")), kw.get("scale_modifier", 1.0), dev(kw.get("cov3D_precomp")),
         dev(kw["viewmatrix"]), dev(kw["projmatrix"])]
    sh = dev(kw.get("shs"))
    empty = torch.Tensor([]).cuda()
    a = [empty if t is None else t for t in a]
    sh = empty if sh is None else sh
    out = C.rasterize_gaussians(*a, kw["tan_fovx"], kw["tan_fovy"], kw["cx"], kw["cy"], kw["H"], kw["W"], sh, 3,
                                dev(kw["campos"]), False, True, False, antialiasing=aa)
    names = ["num_rendered", "n_contrib", "color", "opacity", "depth", "feature", "normal", "surface_xyz", "weights",
             "radii", "geom", "binning", "img"]
    o = dict(zip(names, out))
    S = feats.shape[1]
    o["mid"] = lambda n: C.debug_intermediate(n, P, S, kw["W"], kw["H"], o["geom"], o["img"], o["binning"],
                                              o["num_rendered"])
    if cots is not None:
        extra = {}
        if surface is not None:
            extra["surface"] = (surface[0], surface[1], o["opacity"], o["depth"], kw["cx"], kw["cy"])
            extra["surface_work"] = surface[2]
        g = C.rasterize_gaussians_backward(a[0], a[1], a[2], o["radii"], a[3], a[5], a[6], a[7], a[8], a[9], a[10],
                                           kw["tan_fovx"], kw["tan_fovy"], *[c.contiguous() for c in cots], sh, 3,
                                           dev(kw["campos"]), o["geom"], o["num_rendered"], o["binning"], o["img"],
                                           True, False, antialiasing=aa, absgrad=True, **extra)
        o["grads"], o["absgrad"] = g[:9], g[-1]
    torch.cuda.synchronize()
    return o


@pytest.mark.parametrize("variant", ["plain", "antialiasing", "surface"])
@pytest.mark.parametrize("scene", list(SCENES))
def test_rows_match_fp64_truth(scene, variant):
    kw = SCENES[scene]()
    W, H = kw["W"], kw["H"]
    S = kw["features"].shape[1] if kw.get("features") is not None else 0
    aa = variant == "antialiasing"
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        o = _run(kw, aa=aa)
        P = kw["means3D"].shape[0]
        mid = o["mid"]
        st = dict(point_list=mid("point_list"), ranges=mid("ranges"), n_contrib=mid("n_contrib"),
                  means2D=mid("means2D"), conic_opacity=mid("conic_opacity"), rgb=mid("rgb"), depths=mid("depths"),
                  features=torch.as_tensor(kw["features"]).cuda() if S else torch.zeros(P, 0, device="cuda"))
        bg = torch.as_tensor(kw["bg"]).cuda()
        walks = absgrad64.walks_of(st, W, H)
        amb = torch.zeros(H * W, dtype=torch.bool, device="cuda")
        for wk in walks:
            amb[wk.pix] = wk.ambiguous
        live = (~amb).float().view(1, H, W)
        composited = mid("composited").bool()
        gu = torch.Generator().manual_seed(2)
        unit = [torch.randn(c, H, W, generator=gu).cuda() for c in (3, 1, 1, S)]
        sets = {"unit": unit, "training": _training_cots(o, S, W, H)}
        sets = {k: [c * live for c in cs] for k, cs in sets.items()}
        surf = None
        if variant == "surface":
            ill = torch.as_tensor(surface_oracle.ill_conditioned(o["opacity"], o["depth"], W, H, kw["tan_fovx"],
                                                                 kw["tan_fovy"], kw["cx"], kw["cy"])).cuda()
            # the pull-back reaches the 3x3 neighbours of a normal's pixel: none may reach an ambiguous pixel
            near = torch.nn.functional.max_pool2d((1.0 - live)[None], 3, stride=1, padding=1)[0]
            ok = (~ill).float().view(1, H, W) * (1.0 - near)
            work = torch.empty(_lib.load().r3dg_raster_surface_grad_bytes(W, H, 1), dtype=torch.uint8, device="cuda")
            surf = [torch.randn(3, H, W, generator=gu).cuda() * ok, torch.randn(3, H, W, generator=gu).cuda() * ok, work]
        for sname, cots in sets.items():
            # With the surface cotangents, deterministic mode is not held to the fp64 truth: the pull-back's largest
            # cotangent (up to ~1/opacity at a silhouette) sets the geometry class's fixed-point unit (detacc.cuh),
            # which can then be coarse next to a faint row's terms.  The signed dL_dmeans2D of the same call is
            # printed beside absgrad for comparison.
            if surf is not None:
                torch.use_deterministic_algorithms(True)
                r = _run(kw, cots, aa=aa, surface=surf)
                planes = surf[2][:8 * H * W].view(torch.float32).view(2, 1, H, W)
                ocots = [cots[0], planes[1], planes[0], cots[3]]
                truth, _ = absgrad64.row_truth(st, walks, ocots, bg, W, H, S)
                g64, m = raster64.row_truth(st, walks, ocots, bg, W, H, S)["dL_dmeans2D"]
                ea = ((r["absgrad"].double() - truth).abs() / m.clamp_min(1e-300))[composited]
                es = ((r["grads"][0][:, :2].double() - g64).abs() / m.clamp_min(1e-300))[composited]
                print(f"[absgrad fp64] {scene} surface {sname} det (not asserted): worst / m_row absgrad "
                      f"{float(ea.max()) if ea.numel() else 0.0:.3e}, dL_dmeans2D {float(es.max()) if es.numel() else 0.0:.3e}")
            for mode in ((False,) if surf is not None else (False, True)):
                torch.use_deterministic_algorithms(mode)
                r = _run(kw, cots, aa=aa, surface=surf)
                ocots = cots
                if surf is not None:      # the opacity and depth cotangents the compositor read: the surface pull-back
                    planes = surf[2][:8 * H * W].view(torch.float32).view(2, 1, H, W)     # added (surface_work layout)
                    ocots = [cots[0], planes[1], planes[0], cots[3]]
                truth, _ = absgrad64.row_truth(st, walks, ocots, bg, W, H, S)
                m = raster64.row_truth(st, walks, ocots, bg, W, H, S)["dL_dmeans2D"][1]
                ours = r["absgrad"].double()
                assert bool((r["absgrad"][~composited] == 0).all()) and not bool(
                    torch.signbit(r["absgrad"][~composited]).any()), "rows not composited must be +0"
                keep = composited
                err = (ours - truth).abs()[keep]
                ratio = torch.where(err == 0, torch.zeros_like(err), err / m[keep].clamp_min(1e-300))
                rel = torch.where(err == 0, torch.zeros_like(err), err / truth[keep].clamp_min(1e-300))
                w = float(ratio.max()) if ratio.numel() else 0.0
                print(f"[absgrad fp64] {scene} {variant} {sname} {'det' if mode else 'default'}: worst |g - g64| / m_row "
                      f"{w:.3e} (/ g64 {float(rel.max()) if rel.numel() else 0.0:.3e}) over {int(keep.sum())} rows")
                assert w <= (TAU_AA if aa else TAU[mode]), (scene, variant, sname, mode, w)
    finally:
        torch.use_deterministic_algorithms(prev)


def test_three_views_equal_three_one_view_calls(det):
    P, S = 30_000, 5
    leaves = cg.make_leaves(P, S, seed=4)
    cams = [synth.make_camera(v + 1, W0, H0, center_shift=(v % 2 == 1)) for v in range(3)]
    cots = [cg.cotangents(H0, W0, S, seed=10 + v) for v in range(3)]
    vcot = [torch.stack([c[i] for c in cots]) for i in range(4)]
    _, m_views, _ = _grads(leaves, cams, vcot, V=3, det_mode=True, absgrad=True)
    assert m_views.absgrad.shape == (3, P, 2)
    for v in range(3):
        _, m_one, _ = _grads(leaves, cams[v], cots[v], det_mode=True, absgrad=True)
        assert _bits_equal(m_views.absgrad[v], m_one.absgrad), v


def test_deterministic_reproducible_and_equivariant():
    leaves = cg.make_leaves(P0, 5, seed=5)
    cam = synth.make_camera(2, W0, H0)
    cot = cg.cotangents(H0, W0, 5)
    _, a, _ = _grads(leaves, cam, cot, det_mode=True, absgrad=True)
    _, b, _ = _grads(leaves, cam, cot, det_mode=True, absgrad=True)
    assert _bits_equal(a.absgrad, b.absgrad)
    for k in (1, 8, 21):
        _, c, _ = _grads(leaves, cam, [t * 2.0 ** -k for t in cot], det_mode=True, absgrad=True)
        assert _bits_equal(c.absgrad, a.absgrad * 2.0 ** -k), k


def test_retain_graph_double_backward_doubles(det):
    leaves = cg.make_leaves(P0, 5, seed=6)
    cam = synth.make_camera(3, W0, H0)
    cot = cg.cotangents(H0, W0, 5)
    _, once, _ = _grads(leaves, cam, cot, det_mode=True, absgrad=True)
    _, twice, _ = _grads(leaves, cam, cot, det_mode=True, absgrad=True, twice=True)
    assert _bits_equal(twice.absgrad, once.absgrad * 2)


def test_frozen_means2d_sets_nothing():
    leaves = cg.make_leaves(P0, 5, seed=7)
    leaves = {k: (t.detach() if k not in ("features", "shs") else t) for k, t in leaves.items()}
    cam = synth.make_camera(1, W0, H0)
    vm, pm, cp = cg.camera_tensors(cam, grad=False)
    m2d = torch.zeros(P0, 3, device="cuda")                                # needs no gradient
    other = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
    out = GaussianRasterizer(cg.settings_of(cam, vm, pm, cp), absgrad=True)(leaves["means3D"], m2d,
                                                                             leaves["opacities"], **other)
    sum((out[i] * c).sum() for i, c in zip((2, 3, 4, 5), cg.cotangents(H0, W0, 5))).backward()
    assert not hasattr(m2d, "absgrad")


def test_deferred_overflow_repair_keeps_absgrad(det):
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
        out = GaussianRasterizer(rs, absgrad=True)(leaves["means3D"], m2d, leaves["opacities"], **kw)
        loss = sum((out[i] * c).sum() for i, c in zip((2, 3, 4, 5), cot))
        loss.backward()
        return m2d.absgrad

    cam = synth.make_camera(2, W, H)
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
        assert _bits_equal(got, want)
    finally:
        _C_raster._HEADROOM = old
        set_deferred_count(False)
        _C_raster._state.clear()


def test_densification_uses_the_absgrad_statistic():
    """add_densification_stats(absgrad=True) accumulates |absgrad| where the PyTorch expression does."""
    import densify_oracle as do
    m = do.build_model(do.densify_case("s1_p7"), do.StandIn, device="cuda")
    P = m._xyz.shape[0]
    g = torch.Generator().manual_seed(3)
    vpt = torch.zeros(P, 3, device="cuda", requires_grad=True)
    vpt.grad = torch.randn(P, 3, generator=g).cuda() * 1e-4
    vpt.absgrad = (torch.rand(P, 2, generator=g) * 1e-3).cuda()
    m._normal.grad = torch.randn(P, 3, generator=g).cuda()
    filt = torch.rand(P, generator=g).cuda() > 0.3
    w = torch.rand(P, 1, generator=g).cuda()
    want = m.xyz_gradient_accum.clone()
    want[filt] += torch.norm(vpt.absgrad[filt], dim=-1, keepdim=True)
    densify.add_densification_stats(m, vpt, filt, w, absgrad=True)
    torch.cuda.synchronize()
    assert ((m.xyz_gradient_accum - want).abs() <= 1e-6 * want.abs()).all()
