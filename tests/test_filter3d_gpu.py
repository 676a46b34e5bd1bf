"""Mip-Splatting's 3D filter on the GPU.

compute_3d_filter against the fp64 restatement (tests/filter3d_oracle.py); the filtered rasterizer mode through an
exact decomposition: run A is the mode on with (s, o, f), run B the mode off with fold(s, o, f) = (s', o').  The
forward of A computes exactly B's inputs, so in deterministic mode every forward output and every gradient that does
not pass through the filter is bitwise B's, dL/do = coef dL/do' bit for bit, and dL/ds is the fp64 chain rule applied
to B's dL/ds' and dL/do'.  Also: f = 0 is the mode off, several views, camera / surface / absgrad / frozen-geometry
composition, refusals, sync-freedom and a short training loop."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import filter3d_oracle as fo
from helpers import EDGE_CASES, edge_case
from relightable3dgaussian_b200 import _C_raster, _lib, filter3d, synth
from relightable3dgaussian_b200.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer,
                                                   rasterize_views)

pytestmark = pytest.mark.gpu

GRADS = ("means2D", "colors_precomp", "opacities", "means3D", "features", "cov3D_precomp", "shs", "scales", "rotations",
         "viewmatrix", "projmatrix", "campos")
OUT = ("color", "opacity", "depth", "feature", "normal", "surface_xyz", "weights", "radii", "n_contrib")
# dL/ds against the fp64 chain rule, per entry relative to |dL/ds' s/s'| + |o dL/do' dcoef/ds|: the kernel's chain is
# ~10 correctly rounded fp32 operations on B's fp32 gradients.  An H100 80GB HBM3 (700 W) showed at most 7.0 eps32 over
# every scene below (`shell` with antialiasing); the bound is about twice that.
CHAIN_TAU = 16 * fo.EPS32


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


# ---- compute_3d_filter -------------------------------------------------------------------------------------------

def cameras(V, seed, radius=4.0):
    """V cameras around the origin with mixed focal lengths, principal points and image sizes."""
    g = np.random.default_rng(seed)
    cams = []
    for i in range(V):
        W, H = int(g.integers(64, 900)), int(g.integers(48, 700))
        c = synth.make_camera(i % 8 + 1, W, H, radius=float(radius * g.uniform(0.6, 1.6)))
        fx, fy = float(g.uniform(0.5, 2.0) * W), float(g.uniform(0.5, 2.0) * H)
        cx, cy = float(W * g.uniform(0.3, 0.7)), float(H * g.uniform(0.3, 0.7))
        # a rotation about the camera's own axis keeps it looking at the scene while the V views differ
        a = float(g.uniform(-0.3, 0.3))
        R = torch.tensor([[math.cos(a), -math.sin(a), 0, 0], [math.sin(a), math.cos(a), 0, 0], [0, 0, 1, 0],
                          [0, 0, 0, 1]], dtype=torch.float32)
        wv = (c.viewmatrix.float() @ R).contiguous()
        cams.append(SimpleNamespace(world_view_transform=wv.cuda(), image_width=W, image_height=H, fx=fx, fy=fy, cx=cx,
                                    cy=cy))
    return cams


def oracle_of(means, cams):
    views = torch.stack([c.world_view_transform.cpu() for c in cams]).reshape(len(cams), 16)
    intr = torch.tensor([filter3d._intrinsics(c) + (c.image_width, c.image_height) for c in cams], dtype=torch.float64)
    F = max(r[0] for r in intr.tolist())
    return fo.compute(means.cpu().double(), views.double(), intr, F)


def check_against_oracle(means, cams, report, max_ambiguous=None):
    f = filter3d.compute_3d_filter(means, cams)
    torch.cuda.synchronize()
    assert f.shape == (means.shape[0], 1) and f.dtype == torch.float32
    f64, seen, margin, cond = oracle_of(means, cams)
    amb = margin <= 16                                 # rows with a pair within rounding of a boundary
    report.append(int(amb.sum()))
    limit = max(2, means.shape[0] // 1000) if max_ambiguous is None else max_ambiguous
    assert int(amb.sum()) <= limit, int(amb.sum())
    got = f[:, 0].cpu().double()
    if bool(seen.any()):
        # f = fl(fl(d / F) sqrt(0.2)) with d the fp32 depth (error ~ eps32 times its conditioning), then two roundings;
        # unseen rows take the largest d, which an ambiguous row may have set: only unambiguous seen rows are compared
        tol = 4 * fo.EPS32 * (2 + cond) * f64.abs()
        ok = ~amb & seen
        err = (got - f64).abs()
        assert bool((err[ok] <= tol[ok]).all()), float((err[ok] / tol[ok]).max())
    else:
        assert bool((got == 0).all())
    g = filter3d.compute_3d_filter(means, cams)
    assert bits_equal(f, g)                            # reproducible
    return f


def shell_means(P, seed):
    return synth.make_scene(P, "shell-v1", seed, 0).means3D.float().cuda().contiguous()


@pytest.mark.parametrize("P, V", [(20_000, 1), (20_000, 8), (20_000, 100), (20_000, 300), (1_000_000, 8),
                                  (1_000_000, 100)])
def test_compute_against_fp64(P, V):
    report = []
    check_against_oracle(shell_means(P, 1), cameras(V, V), report)
    print(f"P={P} V={V}: {report[0]} rows within rounding of a boundary")


def test_compute_edges():
    cam = cameras(1, 5)[0]
    M = cam.world_view_transform.cpu().double().reshape(4, 4)      # t = [m, 1] M
    Minv = torch.linalg.inv(M)
    fx, fy, cx, cy = filter3d._intrinsics(cam)
    W, H = cam.image_width, cam.image_height
    pts = []
    for z in (0.2, 0.2 + 1e-6, 0.2 - 1e-6, 1.0, -1.0, -5.0):
        for u, v in ((cx, cy), (-0.15 * W, cy), (1.15 * W, cy), (cx, -0.15 * H), (cx, 1.15 * H), (2 * W, cy)):
            x, y = (u - cx) / fx * z, (v - cy) / fy * z
            pts.append((torch.tensor([x, y, z, 1.0], dtype=torch.float64) @ Minv)[:3])
    means = torch.stack(pts).float().cuda()
    report = []
    check_against_oracle(means, [cam], report, max_ambiguous=len(pts))     # (these rows sit on the boundaries)
    # behind every camera: nothing is seen, f = 0
    behind = means[[i for i in range(len(pts)) if i // 6 >= 4]]
    f = filter3d.compute_3d_filter(behind.contiguous(), [cam])
    assert bool((f == 0).all())
    # P = 0 and P = 1
    assert filter3d.compute_3d_filter(torch.empty(0, 3, device="cuda"), [cam]).shape == (0, 1)
    one = filter3d.compute_3d_filter(means[3:4].contiguous(), [cam])
    assert one.shape == (1, 1) and bool(torch.isfinite(one).all())


def test_compute_is_sync_free_with_a_fixed_launch_count():
    means, cams = shell_means(20_000, 2), cameras(40, 3)
    lib = _lib.load()
    filter3d.compute_3d_filter(means, cams)            # warm up (pinned allocator, library load)
    torch.cuda.synchronize()
    n0 = lib.r3dg_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        filter3d.compute_3d_filter(means, cams)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert lib.r3dg_launch_count() - n0 == 2
    n0 = lib.r3dg_launch_count()
    filter3d.compute_3d_filter(torch.empty(0, 3, device="cuda"), cams)
    assert lib.r3dg_launch_count() == n0


# ---- the filtered rasterizer ---------------------------------------------------------------------------------------

def to_cuda(kw):
    d = {k: (torch.from_numpy(np.ascontiguousarray(v)).float().cuda() if isinstance(v, np.ndarray) else v)
         for k, v in kw.items()}
    if d["opacities"].dim() == 1:
        d["opacities"] = d["opacities"][:, None].contiguous()
    if d.get("features") is None:
        d["features"] = torch.empty(d["means3D"].shape[0], 0, device="cuda")
    return d


def shell_scene():
    sc = synth.make_scene(20_000, "shell-v1", 7, 5)
    cam = synth.make_camera(1, 320, 240)
    d = dict(means3D=sc.means3D, opacities=sc.opacities, viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix,
             campos=cam.campos, bg=torch.tensor([0.1, 0.4, 0.7]), W=cam.image_width, H=cam.image_height,
             tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy, features=sc.features, scale_modifier=1.0,
             shs=sc.shs, scales=sc.scales, rotations=sc.rotations)
    g = torch.Generator().manual_seed(2)
    cots = [torch.randn(c, cam.image_height, cam.image_width, generator=g) for c in (3, 1, 1, 5)]
    d = {k: (v.float().contiguous().cuda() if isinstance(v, torch.Tensor) else v) for k, v in d.items()}
    if d["opacities"].dim() == 1:
        d["opacities"] = d["opacities"][:, None].contiguous()
    return d, [c.cuda() for c in cots]


SCENES = [n for n in EDGE_CASES] + ["shell"]


def scene(name):
    if name == "shell":
        return shell_scene()
    kw, cots = edge_case(name)
    return to_cuda(kw), [torch.from_numpy(c).float().cuda() for c in cots]


def filter_for(d, seed=0, zero_frac=0.2):
    """f per Gaussian from 0 to ~2x its median scale, some exactly 0."""
    P = d["means3D"].shape[0]
    g = torch.Generator().manual_seed(seed)
    med = d["scales"].cpu().median(1).values if d["scales"].numel() else torch.full((P,), 0.01)
    f = med * 2 * torch.rand(P, generator=g)
    f[torch.rand(P, generator=g) < zero_frac] = 0
    return f.float().cuda().contiguous()


def run(d, scales, opac, cots, f=None, aa=False, backward=True, **bkw):
    E = torch.empty(0, device="cuda")
    g = lambda k: d.get(k, E)
    o = _C_raster.rasterize_gaussians(d["bg"], d["means3D"], d["features"], g("colors_precomp"), opac, scales,
                                      g("rotations"), d["scale_modifier"], g("cov3D_precomp"), d["viewmatrix"],
                                      d["projmatrix"], d["tan_fovx"], d["tan_fovy"], d["cx"], d["cy"], d["H"], d["W"],
                                      g("shs"), 3, d["campos"], False, True, False, antialiasing=aa, filter_3d=f)
    r = dict(zip(("num_rendered",) + OUT[-1:] + OUT[:-1], o[:10]))
    if backward:
        kw = dict(bkw)
        if kw.get("geometry", True):
            kw["cam_grads"] = True
        gr = _C_raster.rasterize_gaussians_backward(d["bg"], d["means3D"], d["features"], o[9], g("colors_precomp"),
                                                    scales, g("rotations"), d["scale_modifier"], g("cov3D_precomp"),
                                                    d["viewmatrix"], d["projmatrix"], d["tan_fovx"], d["tan_fovy"],
                                                    *cots, g("shs"), 3, d["campos"], o[10], o[0], o[11], o[12], True,
                                                    False, antialiasing=aa, filter_3d=f,
                                                    opacities=opac if f is not None else None, **kw)
        r["grads"] = dict(zip(GRADS, gr))
    torch.cuda.synchronize()
    return r


def decomposition(d, cots, f, aa, det):
    s, o = d["scales"], d["opacities"]
    A = run(d, s, o, cots, f, aa)
    sf, of = filter3d.fold(s, o, f)
    B = run(d, sf.contiguous(), of.contiguous(), cots, None, aa)
    assert A["num_rendered"] == B["num_rendered"]
    for k in OUT:
        if det or k != "weights":
            assert bits_equal(A[k], B[k]), k
        else:
            torch.testing.assert_close(A[k], B[k], rtol=1e-3, atol=1e-6)
    gA, gB = A["grads"], B["grads"]
    for k in ("means2D", "means3D", "rotations", "shs", "colors_precomp", "features", "viewmatrix", "projmatrix",
              "campos"):
        if gA[k] is None or not gA[k].numel():
            continue
        if det:
            assert bits_equal(gA[k], gB[k]), k
        else:
            assert rel_l2(gA[k], gB[k]) <= 1e-3, (k, rel_l2(gA[k], gB[k]))
    want_do = torch.mul(filter3d_coef(s, f), gB["opacities"][:, 0])
    if det:
        assert bits_equal(gA["opacities"][:, 0], want_do)
    else:
        assert rel_l2(gA["opacities"][:, 0], want_do) <= 1e-3
    ds, _, mag = fo.chain(s, o, f, gB["scales"], gB["opacities"])
    err = (gA["scales"].double() - ds).abs()
    ratio = float((err / mag.clamp_min(1e-300))[mag > 0].max()) if bool((mag > 0).any()) else 0.0
    if det:
        assert ratio <= CHAIN_TAU, ratio / fo.EPS32
    else:
        assert rel_l2(gA["scales"], ds) <= 1e-3
    return A, ratio


def filter3d_coef(s, f):
    """The forward's coef in fp32, in its op order (filter3d.fold's)."""
    f = f.reshape(-1, 1)
    q = s * s
    e = q + f * f
    r = torch.where(e == 0, torch.ones_like(q), q / e)
    return torch.sqrt((r[:, 0] * r[:, 1]) * r[:, 2])


@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
@pytest.mark.parametrize("name", SCENES)
def test_exact_decomposition_deterministic(det_mode, name, aa):
    d, cots = scene(name)
    if "scales" not in d or not d["scales"].numel():
        pytest.skip("scene uses cov3D_precomp")
    _, ratio = decomposition(d, cots, filter_for(d), aa, True)
    print(f"{name} aa={aa}: dL/ds worst ratio {ratio / fo.EPS32:.1f} eps32")


# (`needles` is left to deterministic mode: its dL/dmeans3D is a sum whose terms nearly cancel, so two default-mode runs
# with different float-atomic orders differ by several percent there, with or without the filter)
@pytest.mark.parametrize("name", ["opaque-S5", "inside-x1", "shell"])
def test_decomposition_default_mode(name):
    d, cots = scene(name)
    decomposition(d, cots, filter_for(d, 1), False, False)


@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
@pytest.mark.parametrize("det", [False, True], ids=["default", "det"])
def test_zero_filter_is_the_mode_off(det, aa):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        d, cots = shell_scene()
        z = torch.zeros(d["means3D"].shape[0], device="cuda")
        A = run(d, d["scales"], d["opacities"], cots, z, aa)
        B = run(d, d["scales"], d["opacities"], cots, None, aa)
        for k in OUT:
            if det or k != "weights":
                assert torch.equal(A[k], B[k]), k
        for k in GRADS:
            if A["grads"][k] is not None and A["grads"][k].numel() and det:
                assert torch.equal(A["grads"][k], B["grads"][k]), k
        if not det:
            for k in ("means3D", "scales", "opacities", "shs"):
                assert rel_l2(A["grads"][k], B["grads"][k]) <= 1e-3, k
    finally:
        torch.use_deterministic_algorithms(prev)


def test_large_filter_stays_finite():
    d, cots = shell_scene()
    f = torch.full((d["means3D"].shape[0],), 1e3, device="cuda")
    s = d["scales"].clone()
    s[:10] = 0
    A = run(d, s, d["opacities"], cots, f)
    for k in ("color", "opacity", "depth"):
        assert bool(torch.isfinite(A[k]).all()), k
    for k in ("means3D", "scales", "opacities", "rotations"):
        assert bool(torch.isfinite(A["grads"][k]).all()), k


def test_three_views_equal_one_view_calls(det_mode):
    d, cots = shell_scene()
    f = filter_for(d)
    cams = [synth.make_camera(i, d["W"], d["H"]) for i in (1, 3, 5)]
    P = d["means3D"].shape[0]
    leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "opacities", "scales", "rotations", "shs")}

    def settings(c):
        return GaussianRasterizationSettings(c.image_height, c.image_width, c.tanfovx, c.tanfovy, c.cx, c.cy,
                                             d["bg"], 1.0, c.viewmatrix.cuda(), c.projmatrix.cuda(), 3,
                                             c.campos.cuda(), False, True, True, False)
    m2 = torch.zeros(3, P, 3, device="cuda", requires_grad=True)
    outV = rasterize_views(leaves["means3D"], m2, leaves["opacities"], settings=[settings(c) for c in cams],
                           shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"], filter_3d=f)
    (outV[2] * 0.5).sum().backward()
    gV = {k: v.grad.clone() for k, v in leaves.items()}
    for v in leaves.values():
        v.grad = None
    for i, c in enumerate(cams):
        m1 = torch.zeros(P, 3, device="cuda", requires_grad=True)
        out1 = GaussianRasterizer(settings(c))(means3D=leaves["means3D"], means2D=m1, opacities=leaves["opacities"],
                                               shs=leaves["shs"], scales=leaves["scales"],
                                               rotations=leaves["rotations"], filter_3d=f)
        assert bits_equal(out1[2], outV[2][i])
        (out1[2] * 0.5).sum().backward()
        assert bits_equal(m1.grad, m2.grad[i])
    for k in gV:
        assert rel_l2(gV[k], leaves[k].grad) <= 1e-5, k     # the views' fp32 sum against autograd's sum of three calls


def test_composition_camera_surface_absgrad_frozen():
    d, cots = shell_scene()
    f = filter_for(d)
    cam = synth.make_camera(1, d["W"], d["H"])
    vm = cam.viewmatrix.cuda().requires_grad_(True)
    rs = GaussianRasterizationSettings(d["H"], d["W"], cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, d["bg"], 1.0, vm,
                                       cam.projmatrix.cuda(), 3, cam.campos.cuda(), False, True, True, False)
    leaves = {k: d[k].clone().requires_grad_(True) for k in ("means3D", "opacities", "scales", "rotations", "shs",
                                                            "features")}
    m2 = torch.zeros_like(leaves["means3D"], requires_grad=True)
    out = GaussianRasterizer(rs, surface_grads=True, absgrad=True)(
        means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], shs=leaves["shs"],
        scales=leaves["scales"], rotations=leaves["rotations"], features=leaves["features"], filter_3d=f)
    (out[2].sum() + out[6].square().sum() + out[7].sum()).backward()
    assert vm.grad is not None and bool(torch.isfinite(vm.grad).all()) and float(vm.grad.abs().sum()) > 0
    assert m2.absgrad.shape == (d["means3D"].shape[0], 2) and bool((m2.absgrad >= m2.grad[:, :2].abs() - 1e-6).all())
    # frozen geometry: only the features need a gradient; it equals the full backward's
    feats = d["features"].clone().requires_grad_(True)
    rs2 = rs._replace(viewmatrix=cam.viewmatrix.cuda())
    out2 = GaussianRasterizer(rs2)(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]),
                                   opacities=d["opacities"], shs=d["shs"], scales=d["scales"],
                                   rotations=d["rotations"], features=feats, filter_3d=f)
    out2[5].sum().backward()
    feats_full = d["features"].clone().requires_grad_(True)
    sc = d["scales"].clone().requires_grad_(True)
    out3 = GaussianRasterizer(rs2)(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]),
                                   opacities=d["opacities"], shs=d["shs"], scales=sc, rotations=d["rotations"],
                                   features=feats_full, filter_3d=f)
    out3[5].sum().backward()
    assert rel_l2(feats.grad, feats_full.grad) <= 1e-6


def test_refusals_on_the_device():
    d, _ = shell_scene()
    P = d["means3D"].shape[0]
    cam = synth.make_camera(1, d["W"], d["H"])
    rs = GaussianRasterizationSettings(d["H"], d["W"], cam.tanfovx, cam.tanfovy, cam.cx, cam.cy, d["bg"], 1.0,
                                       cam.viewmatrix.cuda(), cam.projmatrix.cuda(), 3, cam.campos.cuda(), False, True,
                                       True, False)
    R = GaussianRasterizer(rs)
    call = lambda f, **kw: R(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]), opacities=d["opacities"],
                             shs=d["shs"], **({"scales": d["scales"], "rotations": d["rotations"]} | kw), filter_3d=f)
    good = torch.zeros(P, 1, device="cuda")
    for bad in (torch.zeros(P - 1, device="cuda"), torch.zeros(P, 2, device="cuda"), torch.zeros(P),
                torch.zeros(P, device="cuda", dtype=torch.float64), torch.zeros(P, 2, device="cuda")[:, 0],
                torch.zeros(P, device="cuda", requires_grad=True)):
        with pytest.raises(ValueError):
            call(bad)
    with pytest.raises(ValueError, match="cov3D_precomp"):
        R(means3D=d["means3D"], means2D=torch.zeros_like(d["means3D"]), opacities=d["opacities"], shs=d["shs"],
          cov3D_precomp=torch.zeros(P, 6, device="cuda"), filter_3d=good)
    call(good)                                          # the same call with a well-formed filter runs


def test_deferred_count_repair_carries_the_filter(det_mode):
    """Learn the instance counts on small Gaussians, then boost the scales 20x so that the deferred forward overflows
    its binning buffer: the backward re-runs the forward with the filter and gives the synchronous call's gradients."""
    import warnings
    from relightable3dgaussian_b200.rasterizer import set_deferred_count
    P, W, H, S = 3000, 160, 120, 5
    sc = synth.make_scene(P, seed=2, S=S)
    base = {k: getattr(sc, k).cuda().contiguous().requires_grad_(True)
            for k in ("means3D", "opacities", "shs", "scales", "rotations", "features")}
    big = dict(base, scales=(base["scales"].detach() * 20.0).requires_grad_(True))
    f = (sc.scales.median(1).values * torch.rand(P, generator=torch.Generator().manual_seed(3))).cuda().contiguous()
    g = torch.Generator().manual_seed(9)
    cot = [torch.randn(c, H, W, generator=g).cuda() for c in (3, 1, 1, S)]

    def one_view(leaves, cam):
        vm, pm, cp = (t.cuda().contiguous() for t in (cam.viewmatrix, cam.projmatrix, cam.campos))
        rs = GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                           torch.tensor([0.1, 0.4, 0.7], device="cuda"), 1.0, vm, pm, 3, cp, False,
                                           True, True, False)
        m2d = torch.zeros(P, 3, device="cuda", requires_grad=True)
        kw = {k: t for k, t in leaves.items() if k not in ("means3D", "opacities")}
        out = GaussianRasterizer(rs)(leaves["means3D"], m2d, leaves["opacities"], filter_3d=f, **kw)
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
            assert rel_l2(got[k], t) <= 1e-6, k
    finally:
        _C_raster._HEADROOM = old
        set_deferred_count(False)
        _C_raster._state.clear()


def test_training_loop_recomputes_the_filter():
    """500 Adam steps on a synthetic target with the filter recomputed every 100 steps and after each change of P
    (a prune every 150 steps): finite, and the loss ends below where it started."""
    torch.manual_seed(0)
    sc = synth.make_scene(4000, "shell-v1", 3, 0)
    cams = [synth.make_camera(i, 128, 96) for i in range(1, 5)]
    tcams = [SimpleNamespace(world_view_transform=c.viewmatrix.cuda(), image_width=128, image_height=96,
                             FoVx=2 * math.atan(c.tanfovx), FoVy=2 * math.atan(c.tanfovy), fx=None) for c in cams]
    bg = torch.zeros(3, device="cuda")
    target = []
    with torch.no_grad():
        for c in cams:
            rs = GaussianRasterizationSettings(96, 128, c.tanfovx, c.tanfovy, c.cx, c.cy, bg, 1.0, c.viewmatrix.cuda(),
                                               c.projmatrix.cuda(), 3, c.campos.cuda(), False, True, False, False)
            target.append(GaussianRasterizer(rs)(means3D=sc.means3D.cuda(), means2D=torch.zeros(4000, 3, device="cuda"),
                                                 opacities=sc.opacities.cuda().reshape(-1, 1), shs=sc.shs.cuda(),
                                                 scales=sc.scales.cuda(), rotations=sc.rotations.cuda())[2])
    g = torch.Generator().manual_seed(1)
    params = {"xyz": (sc.means3D + 0.05 * torch.randn(sc.means3D.shape, generator=g)).cuda(),
              "log_s": torch.log(sc.scales * 1.5).cuda(), "rot": sc.rotations.cuda(),
              "logit_o": torch.full((4000, 1), 0.0).cuda(), "shs": (sc.shs * 0.5).cuda()}
    params = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    opt = torch.optim.Adam(params.values(), lr=2e-3)
    f = filter3d.compute_3d_filter(params["xyz"].detach(), tcams)
    losses = []
    for it in range(500):
        i = it % len(cams)
        c = cams[i]
        rs = GaussianRasterizationSettings(96, 128, c.tanfovx, c.tanfovy, c.cx, c.cy, bg, 1.0, c.viewmatrix.cuda(),
                                           c.projmatrix.cuda(), 3, c.campos.cuda(), False, True, False, False)
        img = GaussianRasterizer(rs)(means3D=params["xyz"], means2D=torch.zeros_like(params["xyz"]),
                                     opacities=torch.sigmoid(params["logit_o"]), shs=params["shs"],
                                     scales=torch.exp(params["log_s"]), rotations=params["rot"], filter_3d=f)[2]
        loss = (img - target[i]).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
        if it % 150 == 149:                             # prune: P changes, the old filter is stale
            keep = torch.arange(params["xyz"].shape[0], device="cuda") % 50 != 0
            with pytest.raises(ValueError):
                GaussianRasterizer(rs)(means3D=params["xyz"][keep], means2D=torch.zeros_like(params["xyz"][keep]),
                                       opacities=torch.sigmoid(params["logit_o"][keep]), shs=params["shs"][keep],
                                       scales=torch.exp(params["log_s"][keep]), rotations=params["rot"][keep],
                                       filter_3d=f)
            params = {k: v.detach()[keep].clone().requires_grad_(True) for k, v in params.items()}
            opt = torch.optim.Adam(params.values(), lr=2e-3)
            f = filter3d.compute_3d_filter(params["xyz"].detach(), tcams)
        elif it % 100 == 99:
            f = filter3d.compute_3d_filter(params["xyz"].detach(), tcams)
    assert all(math.isfinite(x) for x in losses)
    assert np.mean(losses[-20:]) < np.mean(losses[:20])
