"""The rasterizer's depth statistics on the GPU: on leaves every other output bitwise, depth2 and the median against an
fp64 recomposite on the kernel's own lists, depth2 against the feature-channel form of the reference's depth variance,
the gradients against fp64 autograd, and the flag's composition with the rasterizer's other modes."""
import pytest
import torch

import depthstats64 as ds64
import test_ray_depth_gpu as rdg
from relightable3dgaussian_b200 import _C_raster, synth
from relightable3dgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
NAMES = rdg.NAMES
_bits_equal, _leaves, _settings, _cots = rdg._bits_equal, rdg._leaves, rdg._settings, rdg._cots


def _run(lv, rs, cots=None, det=False, depth_stats=True, means2d_grad=True, **kw):
    """Forward and (with `cots`, which may include "depth2" and "median") backward: (outputs, gradients)."""
    torch.use_deterministic_algorithms(det)
    try:
        P = lv["means3D"].shape[0]
        m2 = torch.zeros(P, 3, device=DEV, requires_grad=means2d_grad)
        out = R.GaussianRasterizer(rs, depth_stats=depth_stats, **kw)(
            means3D=lv["means3D"], means2D=m2, opacities=lv["opacities"], shs=lv["shs"], scales=lv["scales"],
            rotations=lv["rotations"], features=lv["features"])
        assert len(out) == (12 if depth_stats else 10)
        o = dict(zip(NAMES + (("depth2", "median") if depth_stats else ()), out[1:]))
        g = {}
        if cots is not None:
            loss = sum((o[k] * c).sum() for k, c in cots.items())
            leaves = dict(lv, means2D=m2)
            names = [k for k, v in leaves.items() if v.requires_grad]
            gs = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
            g = {k: v for k, v in zip(names, gs) if v is not None}
            if getattr(m2, "absgrad", None) is not None:
                g["absgrad"] = m2.absgrad
        torch.cuda.synchronize()
        return {k: v.detach() for k, v in o.items()}, g
    finally:
        torch.use_deterministic_algorithms(False)


def _stat_cots(W, H, seed=5, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return {"depth2": torch.randn(1, H, W, device=DEV, generator=g) * scale,
            "median": torch.randn(1, H, W, device=DEV, generator=g) * scale}


@pytest.mark.parametrize("ray_depth", [False, True])
@pytest.mark.parametrize("S", list(range(34)))
def test_flag_on_leaves_every_other_output_bitwise(S, ray_depth):
    """All ten outputs bitwise the flag-off call's at every channel group; the gradients (S <= 24, zero cotangents on
    the two new outputs) bitwise in deterministic mode."""
    W, H = 96, 64
    lv = _leaves(500, S, seed=S)
    rs = _settings(synth.make_camera(5, W, H), W, H)
    cots = _cots(W, H, S) if S <= 24 else None
    off, g0 = _run(lv, rs, cots, det=True, depth_stats=False, ray_depth=ray_depth)
    zero = None if cots is None else dict(cots, depth2=torch.zeros(1, H, W, device=DEV),
                                          median=torch.zeros(1, H, W, device=DEV))
    on, g1 = _run(lv, rs, zero, det=True, ray_depth=ray_depth)
    for k in NAMES:
        assert _bits_equal(on[k], off[k]), (S, k)
    assert torch.isfinite(on["depth2"]).all() and torch.isfinite(on["median"]).all()
    for k in g0:
        assert bool((g0[k] == g1[k]).all()), (S, k)


def test_zero_cotangents_without_deterministic_mode_agree_to_atomic_order():
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    rs = _settings(synth.make_camera(2, W, H), W, H)
    cots = _cots(W, H, S)
    _, g0 = _run(lv, rs, cots, depth_stats=False)
    _, g1 = _run(lv, rs, dict(cots, depth2=torch.zeros(1, H, W, device=DEV), median=torch.zeros(1, H, W, device=DEV)))
    for k in g0:
        assert float((g0[k] - g1[k]).norm() / g0[k].norm().clamp_min(1e-30)) <= 1e-5, k


def _kernel_state(lv, rs, W, H, ray_depth):
    """The kernel's forward state for raster64.Walk (lists, n_contrib, records) and its median positions."""
    d = lambda t: t.detach()                                                     # noqa: E731
    out = _C_raster.rasterize_gaussians(rs.bg, d(lv["means3D"]), d(lv["features"]), torch.Tensor([]),
                                        d(lv["opacities"]), d(lv["scales"]), d(lv["rotations"]), 1.0,
                                        torch.Tensor([]), rs.viewmatrix.detach(), rs.projmatrix.detach(), rs.tanfovx,
                                        rs.tanfovy, rs.cx, rs.cy, H, W, d(lv["shs"]), 3, rs.campos.detach(), False,
                                        True, False, ray_depth=ray_depth, depth_stats=True)
    P = lv["means3D"].shape[0]
    geom, binning, img = out[10], out[11], out[12]
    dbg = lambda n: _C_raster.debug_intermediate(n, P, lv["features"].shape[1], W, H, geom, img, binning,  # noqa: E731
                                                 out[0])
    st = dict(means2D=dbg("means2D"), conic_opacity=dbg("conic_opacity"), depths=dbg("depths"),
              point_list=dbg("point_list").long(), ranges=dbg("ranges").long(), n_contrib=out[1])
    return st, out, dbg("median_pos")


@pytest.mark.parametrize("ray_depth", [False, True])
def test_depth2_and_median_against_fp64_recomposite(ray_depth):
    """depth2 to 1e-5 relative, the median depth and its debug position exactly the fp64 rule's, on the kernel's lists;
    pixels whose T before a composited entry lies within fp32 ambiguity of 0.5 (or with an ambiguous alpha decision) are
    excluded and counted (< 1 %)."""
    import raster64
    W, H = 96, 64
    cam = synth.make_camera(1, W, H)
    lv = _leaves(800, 1, seed=4, boost=2.0)
    rs = _settings(cam, W, H)
    st, out, mpos = _kernel_state(lv, rs, W, H, ray_depth)
    wk = raster64.Walk(st, list(range(((W + 15) // 16) * ((H + 15) // 16))), W, H)
    d = st["depths"].double()[wk.ids]
    if ray_depth:
        _, _, _, _, p = rdg._record64(lv, cam, W, H)
        p = p.to(DEV)
        d = d - p[wk.ids, 0] * wk.dx - p[wk.ids, 1] * wk.dy
    d2, med, pos, amb = ds64.walk_stats(wk, d)
    amb = amb | wk.ambiguous | ~wk.nc_ok
    assert float(amb.double().mean()) < 0.01, float(amb.double().mean())
    got2 = out[13].reshape(-1)[wk.pix].double()
    gotm = out[14].reshape(-1)[wk.pix].double()
    gotp = mpos.reshape(-1)[wk.pix].long()
    ok = ~amb
    scale = d2.abs().max()
    assert float(((got2 - d2).abs() / (d2.abs() + 1e-3 * scale))[ok].max()) <= 1e-5
    assert bool((gotp[ok] == pos[ok]).all()), int((gotp[ok] != pos[ok]).sum())
    assert float(((gotm - med).abs() / (med.abs() + 1e-6))[ok].max()) <= 1e-5
    assert bool((gotm[ok & (pos == 0)] == 0).all())


def test_depth2_is_the_reference_feature_channel_with_the_mode_off():
    """Mode off, depth2 is what a depths2 feature channel (tz^2, the reference's render.py) composites, and its
    means3D gradient is that channel's."""
    W, H = 128, 96
    cam = synth.make_camera(3, W, H)
    lv = _leaves(1500, 0, seed=2)
    rs = _settings(cam, W, H)
    V = rs.viewmatrix.detach()
    g2 = _stat_cots(W, H)["depth2"]

    def feature_route():
        z = (torch.cat([lv["means3D"], torch.ones_like(lv["means3D"][:, :1])], 1) @ V)[:, 2:3]
        m2 = torch.zeros_like(lv["means3D"], requires_grad=True)
        out = R.GaussianRasterizer(rs)(means3D=lv["means3D"], means2D=m2, opacities=lv["opacities"], shs=lv["shs"],
                                       scales=lv["scales"], rotations=lv["rotations"], features=z * z)
        (g,) = torch.autograd.grad((out[5] * g2).sum(), lv["means3D"])
        return out[5].detach(), g

    f_img, f_grad = feature_route()
    on, g = _run(lv, rs, {"depth2": g2})
    rel = (on["depth2"] - f_img).abs().max() / f_img.abs().max()
    assert float(rel) <= 1e-6, float(rel)
    relg = (g["means3D"] - f_grad).norm() / f_grad.norm()
    assert float(relg) <= 1e-5, float(relg)


def _render64_stats(lv, cam, W, H, order, nc, mpos, ray_depth):
    """fp64 (depth2, median) of rdg._render64's map on the kernel's lists, the median taken at the kernel's stored
    position (a selection: differentiable through that entry's depth), and the pixels whose T before a composited
    entry is within 1e-5 of 0.5 (ambiguous)."""
    import proj64
    V, Pm = cam["viewmatrix"], cam["projmatrix"]
    m, o, off = lv["means3D"], lv["opacities"].reshape(-1), lv["off"]
    import aa_oracle
    sig = aa_oracle.cov3d_from_six(lv["cov3D"]) if "cov3D" in lv else aa_oracle.cov3d_of(lv["scales"], lv["rotations"])
    t = m @ V[:3, :3] + V[3, :3]
    tx, ty, z = t[:, 0], t[:, 1], t[:, 2]
    hx, hy = W / (2 * cam["tanfovx"]), H / (2 * cam["tanfovy"])
    t0x = proj64._clamp_t(tx, z, 1.3 * cam["tanfovx"])
    t0y = proj64._clamp_t(ty, z, 1.3 * cam["tanfovy"])
    zero = torch.zeros_like(z)
    J = torch.stack([hx / z, zero, -hx * t0x / (z * z), zero, hy / z, -hy * t0y / (z * z)], 1).view(-1, 2, 3)
    T = J @ V[:3, :3].T
    C = T @ sig @ T.transpose(1, 2)
    a, b, c = C[:, 0, 0] + 0.3, C[:, 0, 1], C[:, 1, 1] + 0.3
    det = a * c - b * b
    A, B, Cc = proj64._lin_div(c, det), proj64._lin_div(-b, det), proj64._lin_div(a, det)
    cvec = (T @ (sig @ V[:3, 2])[..., None])[..., 0]
    p = torch.stack([A * cvec[:, 0] + B * cvec[:, 1], B * cvec[:, 0] + Cc * cvec[:, 1]], 1)
    h = m @ Pm[:3, :] + Pm[3, :]
    ndc = h[:, :2] / (h[:, 3:4] + 1e-7) + off[:, :2]
    mean2D = ((ndc + 1.0) * torch.tensor([W, H], dtype=torch.float64, device=m.device) - 1.0) * 0.5
    L = max(1, max(int(x.numel()) for x in order))
    ids = torch.zeros(H * W, L, dtype=torch.long)
    valid = torch.zeros(H * W, L, dtype=torch.bool)
    for pix in range(H * W):
        k = int(nc[pix])
        ids[pix, :k] = order[pix][:k]
        valid[pix, :k] = True
    ids, valid = ids.to(m.device), valid.to(m.device)
    px = torch.arange(H * W, device=m.device)
    x, y = (px % W).double()[:, None], (px // W).double()[:, None]
    dx, dy = mean2D[ids, 0] - x, mean2D[ids, 1] - y
    power = -0.5 * (A[ids] * dx * dx + Cc[ids] * dy * dy) - B[ids] * dx * dy
    alpha = (o[ids] * torch.exp(power)).clamp(max=0.99)
    keep = valid & (power <= 0) & (alpha >= 1.0 / 255.0)
    alpha = torch.where(keep, alpha, torch.zeros_like(alpha))
    Tr = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha[:, :-1]], 1), 1)
    tz = z + off[:, 2]
    d = tz[ids] - p[ids, 0] * dx - p[ids, 1] * dy if ray_depth else tz[ids]
    depth2 = (alpha * Tr * d * d).sum(1)
    k = mpos.reshape(-1).long().to(m.device)
    med = torch.where(k > 0, d.gather(1, (k - 1).clamp_min(0)[:, None])[:, 0], torch.zeros_like(depth2))
    amb = (keep & ((Tr.detach() - 0.5).abs() <= 1e-5)).any(1)
    return depth2.view(1, H, W), med.view(1, H, W), amb.view(H, W)


@pytest.mark.parametrize("kind", ["shell", "clamp", "precomp"])
@pytest.mark.parametrize("ray_depth", [False, True])
@pytest.mark.parametrize("cot", ["unit-depth2", "unit-median", "unit-mixed", "training-scale-mixed"])
@pytest.mark.parametrize("det", [False, True])
def test_gradient_rows_against_fp64(kind, ray_depth, cot, det):
    """Every leaf gradient, per row, against fp64 autograd of the same map on the kernel's lists (rdg._render64's
    conventions), for cotangents on depth2, on the median depth, and both mixed with the existing image outputs."""
    S = 1
    lv, cam, W, H = rdg._row_scene(kind, S)
    P = lv["means3D"].shape[0]
    camt = {k: getattr(cam, k).to(DEV).float().contiguous().requires_grad_(True) for k in ("viewmatrix", "projmatrix")}
    rs = R.GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                         torch.tensor([0.1, 0.2, 0.3], device=DEV), 1.0, camt["viewmatrix"],
                                         camt["projmatrix"], 0, cam.campos.to(DEV), False, True, True, False)
    dev = {k: v.to(DEV).float().contiguous() for k, v in lv.items()}
    order, nc = rdg._lists_of(rs, dev, W, H)
    leaf_names = ["means3D", "opacities"] + (["cov3D"] if "cov3D" in lv else ["scales", "rotations"])
    leaves = {k: dev[k].clone().requires_grad_(True) for k in leaf_names}
    m2 = torch.zeros(P, 3, device=DEV, requires_grad=True)
    torch.use_deterministic_algorithms(det)
    try:
        o = R.GaussianRasterizer(rs, ray_depth=ray_depth, depth_stats=True)(
            means3D=leaves["means3D"], means2D=m2, opacities=leaves["opacities"], colors_precomp=dev["colors"],
            scales=leaves.get("scales"), rotations=leaves.get("rotations"), cov3D_precomp=leaves.get("cov3D"),
            features=dev["features"])
    finally:
        torch.use_deterministic_algorithms(False)
    mpos = _C_raster.debug_intermediate("median_pos", P, S, W, H, *_buffers_of(o)).cpu()
    lv64 = {k: v.to(DEV).double().requires_grad_(True) for k, v in lv.items()}
    lv64["off"] = torch.zeros(P, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    cam64 = dict(viewmatrix=cam.viewmatrix.to(DEV).double().requires_grad_(True),
                 projmatrix=cam.projmatrix.to(DEV).double().requires_grad_(True), tanfovx=cam.tanfovx,
                 tanfovy=cam.tanfovy)
    out64, amb = rdg._render64(lv64, cam64, W, H, order, nc, rs.bg.double(), ray_depth)
    d2_64, med64, amb2 = _render64_stats(lv64, cam64, W, H, order, nc, mpos, ray_depth)
    amb = amb | amb2
    assert float(amb.double().mean()) < 0.05
    scale = 2.0 ** -21 if cot.startswith("training") else 1.0
    cots = _stat_cots(W, H, scale=scale)
    if cot == "unit-depth2":
        cots.pop("median")
    elif cot == "unit-median":
        cots.pop("depth2")
    else:
        cots.update(_cots(W, H, S, scale=scale))
    cots = {k: c * (~amb).float() for k, c in cots.items()}
    out64 = dict(out64, depth2=d2_64, median=med64)
    loss = sum((out64[k] * c.double()).sum() for k, c in cots.items())
    wrt = [lv64[k] for k in leaf_names] + [lv64["off"], cam64["viewmatrix"], cam64["projmatrix"]]
    # (a median-only loss does not depend on the opacities: their truth is zero)
    want = [torch.zeros_like(x) if g is None else g
            for x, g in zip(wrt, torch.autograd.grad(loss, wrt, allow_unused=True))]
    img = dict(color=o[2], opacity=o[3], depth=o[4], feature=o[5], depth2=o[10], median=o[11])
    torch.use_deterministic_algorithms(det)
    try:
        loss32 = sum((img[k] * c).sum() for k, c in cots.items())
        got = torch.autograd.grad(loss32, [leaves[k] for k in leaf_names] + [m2, camt["viewmatrix"],
                                                                             camt["projmatrix"]])
    finally:
        torch.use_deterministic_algorithms(False)
    tau = 2e-3
    for k, g32, g64 in zip(leaf_names + ["means2D"], got, want):
        _row_check(g32, g64, tau, (kind, k))
    rdg._row_check(got[-2].view(4, 4)[:, :3].reshape(1, -1), want[-2].view(4, 4)[:, :3].reshape(1, -1), tau,
                   (kind, "viewmatrix"))
    rdg._row_check(got[-1].view(4, 4)[:, [0, 1, 3]].reshape(1, -1), want[-1].view(4, 4)[:, [0, 1, 3]].reshape(1, -1),
                   tau, (kind, "projmatrix"))


def _row_check(got, want, tau, what):
    """rdg._row_check with the row scale floored at 1e-4 of the leaf's largest |g64| (not 1e-6): depth2's cotangent
    enters dL/dalpha as d^2 g2, so a row whose terms cancel to a small total carries fp32 rounding of terms ~d^2 larger
    than the total (the one-scalar A recurrence of the backward, composite_bwd.cu)."""
    got, want = got.double().reshape(want.shape[0], -1), want.reshape(want.shape[0], -1)
    scale = want.abs().amax(1, keepdim=True) + 1e-4 * want.abs().max()
    r = (got - want).abs() / scale.clamp_min(1e-300)
    bad = (r > tau).any(1)
    assert not bool(bad.any()), (what, int(bad.sum()), float(r.max()))


def _buffers_of(outputs):
    """(geomBuffer, imgBuffer, binningBuffer) of a GaussianRasterizer call, from its autograd node's saved tensors."""
    saved = outputs[2].grad_fn.saved_tensors
    return saved[8], saved[10], saved[9]


def test_several_views_are_their_one_view_calls():
    W, H, S = 96, 64, 5
    lv = _leaves(1200, S)
    cams = [synth.make_camera(v, W, H) for v in (0, 3)]
    settings = [_settings(c, W, H) for c in cams]
    cots = [dict(_cots(W, H, S, seed=v), **_stat_cots(W, H, seed=10 + v)) for v in range(2)]
    torch.use_deterministic_algorithms(True)
    try:
        m2 = torch.zeros(2, lv["means3D"].shape[0], 3, device=DEV, requires_grad=True)
        out = R.rasterize_views(lv["means3D"], m2, lv["opacities"], settings=settings, shs=lv["shs"],
                                scales=lv["scales"], rotations=lv["rotations"], features=lv["features"],
                                depth_stats=True)
        names = NAMES + ("depth2", "median")
        loss = sum((dict(zip(names, out[1:]))[k][v] * c).sum() for v in range(2) for k, c in cots[v].items())
        (gv,) = torch.autograd.grad(loss, [lv["means3D"]])
    finally:
        torch.use_deterministic_algorithms(False)
    g1 = 0
    for v in range(2):
        o, g = _run(lv, settings[v], cots[v], det=True)
        for k in ("depth2", "median"):
            assert _bits_equal(dict(zip(NAMES + ("depth2", "median"), out[1:]))[k][v], o[k]), (v, k)
        g1 = g["means3D"] if v == 0 else g1 + g["means3D"]
    assert _bits_equal(gv, g1)


def test_deterministic_mode_is_reproducible():
    W, H, S = 160, 120, 5
    lv = _leaves(2000, S)
    rs = _settings(synth.make_camera(2, W, H), W, H)
    cots = dict(_cots(W, H, S), **_stat_cots(W, H))
    for rd in (False, True):
        o0, g0 = _run(lv, rs, cots, det=True, ray_depth=rd)
        o1, g1 = _run(lv, rs, cots, det=True, ray_depth=rd)
        for k in o0:
            assert _bits_equal(o0[k], o1[k]), (rd, k)
        for k in g0:
            assert _bits_equal(g0[k], g1[k]), (rd, k)


def test_deterministic_scale_at_the_depth_bound():
    """The geometry class's exponent takes |g2| max(Z^2, 2 Z) (Z: the largest |d| of an accepted entry).  At a depth2
    cotangent that puts that product within 2^5 of 2^101, where the exponent reaches its clamp (R3DG_DET_SCALE_MAX = 100),
    the sums are still exact: the gradients are bitwise 2^k times those of the unit cotangent, run to run."""
    W, H, S = 96, 64, 0
    lv = _leaves(800, S, seed=9)
    rs = _settings(synth.make_camera(1, W, H), W, H)
    V = rs.viewmatrix.detach()
    z = (torch.cat([lv["means3D"].detach(), torch.ones_like(lv["means3D"][:, :1])], 1) @ V)[:, 2]
    zmax = float(z.abs().max())                      # >= Z (mode off: d = tz of the accepted entries)
    g2 = torch.sign(_stat_cots(W, H)["depth2"])      # |g2| = 1
    k = 96 - int(torch.ceil(torch.log2(torch.tensor(max(zmax * zmax, 2 * zmax)))))
    assert k > 60
    _, g_unit = _run(lv, rs, {"depth2": g2}, det=True)
    _, g_big = _run(lv, rs, {"depth2": g2 * 2.0 ** k}, det=True)
    _, g_big2 = _run(lv, rs, {"depth2": g2 * 2.0 ** k}, det=True)
    for key in g_unit:
        assert torch.isfinite(g_big[key]).all(), key
        assert _bits_equal(g_big[key], g_big2[key]), key
        assert _bits_equal(g_big[key], g_unit[key] * 2.0 ** k), key


def test_frozen_geometry_gets_the_flag_off_appearance_gradients():
    W, H, S = 128, 96, 5
    lv = {k: v.detach().requires_grad_(k in ("shs", "features")) for k, v in _leaves(1500, S).items()}
    rs = _settings(synth.make_camera(1, W, H), W, H)
    cots = dict(_cots(W, H, S), **_stat_cots(W, H))
    _, g0 = _run(lv, rs, {k: v for k, v in cots.items() if k not in ("depth2", "median")}, det=True,
                 depth_stats=False, means2d_grad=False)
    _, g1 = _run(lv, rs, cots, det=True, means2d_grad=False)
    assert set(g0) == set(g1) == {"shs", "features"}
    for k in g0:
        assert _bits_equal(g0[k], g1[k]), k


@pytest.mark.parametrize("det", [False, True])
def test_absgrad_bounds_the_signed_gradient(det):
    W, H, S = 128, 96, 5
    lv = _leaves(1500, S)
    rs = _settings(synth.make_camera(1, W, H), W, H)
    for rd in (False, True):
        _, g = _run(lv, rs, dict(_cots(W, H, S), **_stat_cots(W, H)), det=det, absgrad=True, ray_depth=rd)
        assert bool((g["absgrad"] >= g["means2D"][:, :2].abs() * (1 - 1e-5)).all()), rd


@pytest.mark.parametrize("variant", ["antialiasing", "filter_3d", "surface_grads"])
def test_composes_with_the_other_modes(variant):
    W, H, S = 128, 96, 5
    lv = _leaves(1500, S)
    rs = _settings(synth.make_camera(1, W, H), W, H)
    kw = {"antialiasing": {"antialiasing": True}, "surface_grads": {"surface_grads": True},
          "filter_3d": {}}[variant]
    if variant == "filter_3d":
        f3d = torch.full((lv["means3D"].shape[0],), 0.01, device=DEV)
        out = R.GaussianRasterizer(rs, depth_stats=True)(
            means3D=lv["means3D"], means2D=torch.zeros_like(lv["means3D"]), opacities=lv["opacities"],
            shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"], features=lv["features"], filter_3d=f3d)
        off = R.GaussianRasterizer(rs)(
            means3D=lv["means3D"], means2D=torch.zeros_like(lv["means3D"]), opacities=lv["opacities"],
            shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"], features=lv["features"], filter_3d=f3d)
        loss = (out[10] * _stat_cots(W, H)["depth2"]).sum() + out[4].sum()
        (g,) = torch.autograd.grad(loss, [lv["scales"]])
        assert torch.isfinite(g).all() and float(g.abs().sum()) > 0
        for i in (1, 2, 3, 4, 5, 6, 7, 9):          # (out_weights: float atomics)
            assert torch.equal(out[i], off[i]), i
        return
    cots = dict(_cots(W, H, S), **_stat_cots(W, H))
    on, g1 = _run(lv, rs, cots, det=True, **kw)
    off, _ = _run(lv, rs, None, det=True, depth_stats=False, **kw)
    for k in NAMES:
        assert _bits_equal(on[k], off[k]), (variant, k)
    for k, v in g1.items():
        assert torch.isfinite(v).all(), (variant, k)


def test_deferred_count_repair_reruns_the_forward_with_the_flag(monkeypatch):
    """A deferred forward whose binning buffer overflowed is re-run in the backward with the flag, and the gradients
    equal the synchronous call's."""
    W, H, S = 128, 96, 5
    lv = _leaves(1500, S)
    rs = _settings(synth.make_camera(1, W, H), W, H)
    cots = dict(_cots(W, H, S), **_stat_cots(W, H))
    _, want = _run(lv, rs, cots, det=True)
    calls = []
    real = _C_raster.rasterize_gaussians

    def tiny(*args, **kw):
        calls.append(kw)
        if kw.get("_defer"):
            kw["_min_capacity"] = 64                 # force the overflow of the deferred attempt
        return real(*args, **kw)
    monkeypatch.setattr(R._C, "rasterize_gaussians", tiny)
    monkeypatch.setattr(_C_raster, "_LEARN", 0)
    R.set_deferred_count(True)
    try:
        with pytest.warns(UserWarning):
            _, got = _run(lv, rs, cots, det=True)
    finally:
        R.set_deferred_count(False)
    assert any(k.get("_defer") for k in calls) and calls[-1].get("depth_stats") is True
    for k in want:
        assert _bits_equal(got[k], want[k]), k
