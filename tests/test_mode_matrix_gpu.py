"""Every backward-compositor instantiation and every composition of the rasterizer's modes against one fp64 truth,
render64 (autograd of the whole map on the kernel's own lists).

(a) The compositor matrix: S in CHANNELS (channel groups NG = 1..7, both sides of the switch from 16 to 8 entries per
    sub-batch) crossed with KERNELS, the (DET, GEOM, ABS, RD, DS) tuples launch_bwd_ng dispatches.
(b) Mode compositions: the projection's modes (none, antialiasing, 3D filter, both) crossed with the compositor's
    (ray depth, depth statistics, surface gradients and their combinations, absgrad) on three scenes, in both modes.
(c) Long lists: tiles of more than 2048 entries and pixels of several hundred contributors, at NG = 7.
(d) Several views in one rasterize_views call.

Each case checks every leaf gradient, means2D, absgrad where on, and the camera's, per row:
|g - g64| <= TAU (max_row |g64| + f max |g64|), f = 1e-6, or 1e-4 with a depth2 cotangent (test_depth_stats_gpu's
_row_check gives the reason), at unit and training-scale (2^-21) cotangents.  Pixels whose fp32 decisions the fp64
truth may take the other way get zero cotangents in both calls, and are fewer than 5 %.

An opacity row may instead meet the compositor's own bound |g - g64| <= TAU_ROW m_row (test_det_scale_gpu.TAU, m_row
the sum of the magnitudes of the row's per-pixel terms, render64.opacity_magnitude).  dL/do = sum over pixels of
dL/dalpha G, and dL/dalpha is a difference the backward forms in fp32 from the colour behind the entry and the
accumulated colour; a Gaussian whose pull on the image is balanced sums such terms to a total far below each of them.
On an H100 (80 GB HBM3, 700 W) the first run of this file found three such rows, one row each in (a) S = 18 plain
and (b) shell surface and shell 3D filter + ray depth: 6.5e-3, 2.3e-3 and 1.8e-2 of max_row |g64|, but 6.4e-7,
4.7e-6 and 6.6e-7 of m_row, fp32 rounding of terms that cancel.  They are identical in both modes, so the error is in
the fp32 terms, not in the order of their sum.  Every other row of every case meets the first bound."""
import functools
import math

import pytest
import torch

import render64
import test_ray_depth_gpu as rdg
from test_det_scale_gpu import TAU as TAU_ROW
from relightable3dgaussian_b200 import _C_raster, synth
from relightable3dgaussian_b200 import rasterizer as R

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")

CHANNELS = (1, 5, 6, 13, 17, 18, 24)
# (GEOM, ABS, RD, DS): the nine flag sets of launch_bwd_ng (GEOM off: the appearance-only backward)
_FLAG_SETS = ((False, False, False, False), (True, False, False, False), (True, True, False, False),
              (True, False, True, False), (True, True, True, False), (True, False, False, True),
              (True, True, False, True), (True, False, True, True), (True, True, True, True))
KERNELS = tuple((det,) + f for det in (False, True) for f in _FLAG_SETS)          # (DET, GEOM, ABS, RD, DS)
TAU = 2e-3
SCALES = (("unit", 1.0), ("training-scale", 2.0 ** -21))
GEOMETRY = ("means3D", "opacities", "scales", "rotations", "cov3D")
APPEARANCE = ("colors", "shs", "features")


def _kid(k):
    return "det" if k[0] else "default", "-".join(n for n, on in zip(("geom", "abs", "rd", "ds"), k[1:]) if on) or "app"


# ---- scenes ---------------------------------------------------------------------------------------------------------
class Scene:
    """Leaves (fp32, on the GPU), camera and image size; D > 0: SH colours, and campos gets a gradient."""

    def __init__(self, leaves, cam, W, H, D=0, filter_3d=None, bg=(0.1, 0.2, 0.3)):
        self.lv = {k: v.to(DEV).float().contiguous() for k, v in leaves.items()}
        self.cam, self.W, self.H, self.D = cam, W, H, D
        self.f3d = filter_3d
        self.bg = torch.tensor(bg, device=DEV)
        self.P = self.lv["means3D"].shape[0]
        self.S = self.lv["features"].shape[1]


def _row_scene(kind, S, sh=False):
    lv, cam, W, H = rdg._row_scene(kind, S)
    D = 0
    if sh:
        g = torch.Generator().manual_seed(17)
        P = lv["means3D"].shape[0]
        shs = 0.25 * torch.randn(P, 16, 3, generator=g)
        shs[:, 0] = (lv.pop("colors") - 0.5) / 0.28209479177387814
        lv["shs"], D = shs, 3
    return lv, cam, W, H, D


def _filter_3d(P):
    g = torch.Generator().manual_seed(3)
    f = 0.002 + 0.01 * torch.rand(P, generator=g)
    f[::3] = 0.0
    return f.to(DEV).contiguous()


# ---- the kernel -----------------------------------------------------------------------------------------------------
def _settings(sc, V=None, P=None, campos=None):
    c = sc.cam
    return R.GaussianRasterizationSettings(sc.H, sc.W, c.tanfovx, c.tanfovy, c.cx, c.cy, sc.bg, 1.0, V, P, sc.D,
                                           campos, False, True, True, False)


def _image_dict(out, ds):
    o = dict(color=out[2], opacity=out[3], depth=out[4], feature=out[5], normal=out[6], xyz=out[7])
    if ds:
        o.update(depth2=out[10], median=out[11])
    return o


def _inputs(sc, grads):
    lv = {k: v.clone().requires_grad_(k in grads) for k, v in sc.lv.items()}
    return lv, dict(shs=lv.get("shs"), colors_precomp=lv.get("colors"), scales=lv.get("scales"),
                    rotations=lv.get("rotations"), cov3D_precomp=lv.get("cov3D"), features=lv["features"])


def _state(sc, aa, rd):
    """The forward state render64 walks (the lists, n_contrib, the kernel's means2D and conic, median_pos, clamped)."""
    cam = [getattr(sc.cam, k).to(DEV).float().contiguous() for k in ("viewmatrix", "projmatrix", "campos")]
    lv, kw = _inputs(sc, ("means3D",))
    m2 = torch.zeros(sc.P, 3, device=DEV)
    out = R.GaussianRasterizer(_settings(sc, *cam), antialiasing=aa, ray_depth=rd, depth_stats=True)(
        means3D=lv["means3D"], means2D=m2, opacities=lv["opacities"], filter_3d=sc.f3d, **kw)
    saved = out[2].grad_fn.saved_tensors
    geom, binning, img = saved[8], saved[9], saved[10]
    mid = lambda n: _C_raster.debug_intermediate(n, sc.P, sc.S, sc.W, sc.H, geom, img, binning, out[0])  # noqa: E731
    st = dict(point_list=mid("point_list").long(), ranges=mid("ranges").long(), n_contrib=out[1].detach(),
              means2D=mid("means2D"), conic_opacity=mid("conic_opacity"), median_pos=mid("median_pos"))
    return st, mid("clamped").double()


def _kernel(sc, mode, cots, det):
    """One forward and backward of GaussianRasterizer in `mode` with cotangents `cots`: {name: gradient}."""
    geom = mode.get("geom", True)
    grads = (GEOMETRY + APPEARANCE) if geom else APPEARANCE
    lv, kw = _inputs(sc, grads)
    cam = {k: getattr(sc.cam, k).to(DEV).float().contiguous().requires_grad_(geom and (k != "campos" or sc.D > 0))
           for k in ("viewmatrix", "projmatrix", "campos")}
    m2 = torch.zeros(sc.P, 3, device=DEV, requires_grad=geom)
    torch.use_deterministic_algorithms(det)
    try:
        out = R.GaussianRasterizer(_settings(sc, cam["viewmatrix"], cam["projmatrix"], cam["campos"]),
                                   surface_grads=mode.get("surf", False), antialiasing=mode.get("aa", False),
                                   absgrad=mode.get("abs", False), ray_depth=mode.get("rd", False),
                                   depth_stats=mode.get("ds", False))(
            means3D=lv["means3D"], means2D=m2, opacities=lv["opacities"], filter_3d=sc.f3d, **kw)
        img = _image_dict(out, mode.get("ds", False))
        loss = sum((img[k] * c).sum() for k, c in cots.items())
        wrt = {k: v for k, v in lv.items() if v.requires_grad}
        wrt.update({k: v for k, v in cam.items() if v.requires_grad})
        if geom:
            wrt["means2D"] = m2
        g = dict(zip(wrt, torch.autograd.grad(loss, list(wrt.values()), allow_unused=True)))
        if mode.get("abs", False):
            g["absgrad"] = m2.absgrad
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    return {k: v for k, v in g.items() if v is not None}


# ---- the truth ------------------------------------------------------------------------------------------------------
def _cam64(sc, cam=None):
    c = sc.cam if cam is None else cam
    t = {k: getattr(c, k).to(DEV).double().contiguous().requires_grad_(True)
         for k in ("viewmatrix", "projmatrix", "campos")}
    return t, render64.Camera(t["viewmatrix"], t["projmatrix"], t["campos"], sc.W, sc.H, c.tanfovx, c.tanfovy, c.cx,
                              c.cy)


def _truth(sc, mode, st, clamped, seed=1, cam=None):
    """(cotangents, {name: g64}, ambiguous fraction, render) of `mode` at unit cotangents (zero on ambiguous pixels)."""
    lv = {k: v.double().requires_grad_(True) for k, v in sc.lv.items()}
    lv["off"] = torch.zeros(sc.P, 3, dtype=torch.float64, device=DEV, requires_grad=True)
    ct, cam64 = _cam64(sc, cam)
    const = {"clamped": clamped}
    if sc.f3d is not None:
        const["filter_3d"] = sc.f3d.double()
    out = render64.render(lv, const, cam64, st, sc.bg.double(), D=sc.D, aa=mode.get("aa", False),
                          f3d=sc.f3d is not None, ray_depth=mode.get("rd", False), depth_stats=mode.get("ds", False),
                          surface=mode.get("surf", False), batch_pixels=mode.get("batch_pixels", 1 << 14))
    amb = out.ambiguous_pixels()
    live = (~amb).float()[None]
    g = torch.Generator(device=DEV).manual_seed(seed)
    names = ["color", "opacity", "depth", "feature"] + (["depth2", "median"] if mode.get("ds") else []) + \
        (["normal", "xyz"] if mode.get("surf") else [])
    cots = {k: torch.randn(out.images[k].shape, device=DEV, generator=g) * live for k in names}
    loss = sum((out.images[k] * c.double()).sum() for k, c in cots.items())
    wrt = dict(lv, **ct)
    if sc.D == 0:
        wrt.pop("campos")
    gs = torch.autograd.grad(loss, list(wrt.values()) + out.pair_leaves(), allow_unused=True)
    want = {k: torch.zeros_like(v) if gg is None else gg for (k, v), gg in zip(wrt.items(), gs)}
    want["means2D"] = want.pop("off")
    want["absgrad"] = out.absgrad(gs[len(wrt):])
    want["opacities_mrow"] = out.opacity_magnitude(gs[len(wrt):])
    return cots, want, float(amb.double().mean()), out


def _row_errors(got, want, floor):
    """Per row: max |g - g64| / (max_row |g64| + floor max |g64|) (rdg._row_check's ratio)."""
    got, want = got.double().reshape(want.shape[0], -1), want.reshape(want.shape[0], -1)
    scale = want.abs().amax(1, keepdim=True) + floor * want.abs().max()
    return ((got - want).abs() / scale.clamp_min(1e-300)).amax(1)


def _compare(got, want, scale, floor, what, fails, names=None):
    """Every gradient `got` holds (or `names`) against want * scale; failures appended as (what, name, rows, worst)."""
    for k in (names or got):
        if k not in want:
            continue
        g, w = got[k], want[k] * scale
        if k == "viewmatrix":
            g, w = g.reshape(-1, 4, 4)[:, :, :3].reshape(-1, 12), w.reshape(-1, 4, 4)[:, :, :3].reshape(-1, 12)
        elif k == "projmatrix":
            g, w = (g.reshape(-1, 4, 4)[:, :, [0, 1, 3]].reshape(-1, 12),
                    w.reshape(-1, 4, 4)[:, :, [0, 1, 3]].reshape(-1, 12))
        elif k == "campos":
            g, w = g.reshape(-1, 3), w.reshape(-1, 3)
        r = _row_errors(g, w, floor)
        if k == "opacities" and "opacities_mrow" in want:
            e = (g.double().reshape(-1) - w.reshape(-1)).abs() / (want["opacities_mrow"] * scale).clamp_min(1e-300)
            within = e <= TAU_ROW
            if bool(((r > TAU) & within).any()):
                print(f"[opacity rows] {what}: {int(((r > TAU) & within).sum())} row(s) within TAU_ROW m_row, "
                      f"|g - g64| / row scale {float(r[(r > TAU) & within].max()):.3e}, "
                      f"/ m_row {float(e[(r > TAU) & within].max()):.3e}")
            r = torch.where(within, torch.zeros_like(r), r)
        worst = float(r.max()) if r.numel() else 0.0
        if worst > TAU or not math.isfinite(worst):
            fails.append((what, k, int((r > TAU).sum()), worst))


def _run_case(sc, mode, want, cots, fails, what, names=None, dets=(False, True)):
    floor = 1e-4 if "depth2" in cots else 1e-6
    for det in dets:
        for sname, s in SCALES:
            got = _kernel(sc, mode, {k: c * s for k, c in cots.items()}, det)
            _compare(got, want, s, floor, (what, "det" if det else "default", sname), fails, names)
            if names is None:
                missing = set(got) - set(want)
                assert not missing, missing


# ---- (a) the compositor matrix --------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def _matrix_truth(S, rd, ds):
    lv, cam, W, H, D = _row_scene("shell", S)
    sc = Scene(lv, cam, W, H, D)
    st, clamped = _state(sc, False, rd)
    cots, want, amb, _ = _truth(sc, dict(rd=rd, ds=ds), st, clamped)
    return sc, cots, want, amb


@pytest.mark.parametrize("kernel", KERNELS, ids=lambda k: "-".join(_kid(k)))
@pytest.mark.parametrize("S", CHANNELS)
def test_compositor_matrix(S, kernel):
    det, geom, ab, rd, ds = kernel
    sc, cots, want, amb = _matrix_truth(S, rd, ds)
    assert amb < 0.05, amb
    mode = dict(geom=geom, abs=ab, rd=rd, ds=ds)
    fails = []
    names = None if geom else ("colors", "features")
    if not geom:
        cots = {k: c for k, c in cots.items() if k in ("color", "feature")}
    _run_case(sc, mode, want, cots, fails, (S,) + _kid(kernel), names=names, dets=(det,))
    assert not fails, fails


# ---- (b) mode compositions ------------------------------------------------------------------------------------------
PROJ_MODES = {"plain": {}, "aa": {"aa": True}, "f3d": {"f3d": True}, "aa+f3d": {"aa": True, "f3d": True}}
COMP_MODES = {"rd": {"rd": True}, "ds": {"ds": True}, "rd+ds+abs": {"rd": True, "ds": True, "abs": True},
              "surf": {"surf": True}, "surf+rd": {"surf": True, "rd": True},
              "surf+rd+ds+abs": {"surf": True, "rd": True, "ds": True, "abs": True}}


@pytest.mark.parametrize("comp", list(COMP_MODES))
@pytest.mark.parametrize("proj", list(PROJ_MODES))
@pytest.mark.parametrize("kind", ["shell", "clamp", "precomp"])
def test_mode_compositions(kind, proj, comp):
    mode = dict(PROJ_MODES[proj], **COMP_MODES[comp])
    lv, cam, W, H, D = _row_scene(kind, 5, sh=(kind == "shell"))
    f3d = _filter_3d(lv["means3D"].shape[0]) if mode.get("f3d") else None
    sc = Scene(lv, cam, W, H, D, filter_3d=f3d)
    if f3d is not None and "cov3D" in lv:
        with pytest.raises(ValueError):
            _kernel(sc, mode, {}, False)
        return
    st, clamped = _state(sc, mode.get("aa", False), mode.get("rd", False))
    cots, want, amb, _ = _truth(sc, mode, st, clamped)
    assert amb < 0.05, amb
    fails = []
    _run_case(sc, mode, want, cots, fails, (kind, proj, comp))
    assert not fails, fails


# ---- (c) long lists -------------------------------------------------------------------------------------------------
def _long_scene():
    """3000 faint Gaussians (opacity 0.02-0.06) of 6-14 px screen sigma, centred around the image centre."""
    W, H, P, S = 96, 64, 3000, 24
    cam = synth.make_axis_camera(W, H)
    g = torch.Generator().manual_seed(21)
    f = W / (2 * cam.tanfovx)
    z = 3.0 + 2.0 * torch.rand(P, generator=g)
    u = 48.0 + 18.0 * torch.randn(P, generator=g)
    v = 32.0 + 12.0 * torch.randn(P, generator=g)
    x, y = (u + 0.5 - W / 2) / f * z, (v + 0.5 - H / 2) / f * z
    sig = (6.0 + 8.0 * torch.rand(P, generator=g)) * z / f
    scales = sig[:, None] * (0.7 + 0.6 * torch.rand(P, 3, generator=g))
    q = torch.randn(P, 4, generator=g)
    lv = dict(means3D=torch.stack([x, y, z], 1), opacities=(0.02 + 0.04 * torch.rand(P, 1, generator=g)),
              colors=torch.rand(P, 3, generator=g), scales=scales, rotations=q / q.norm(dim=1, keepdim=True),
              features=torch.rand(P, S, generator=g))
    return Scene(lv, cam, W, H)


def test_long_lists():
    sc = _long_scene()
    mode = dict(aa=True, rd=True, ds=True, abs=True, batch_pixels=2048)
    st, clamped = _state(sc, True, True)
    tile_len = (st["ranges"][:, 1] - st["ranges"][:, 0]).max()
    print(f"[long lists] longest tile list {int(tile_len)}, most contributors {int(st['n_contrib'].max())}")
    assert int(tile_len) > 2048                 # the backward refills its mask stream, the forward runs many batches
    assert int(st["n_contrib"].max()) >= 300    # several sub-batches per walk
    cots, want, amb, _ = _truth(sc, mode, st, clamped)
    print(f"[long lists] ambiguous pixels {amb:.4f}")
    assert amb < 0.05, amb
    fails = []
    _run_case(sc, mode, want, cots, fails, "long lists")
    assert not fails, fails


# ---- (d) several views ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("det", [False, True])
def test_several_views(det):
    """One rasterize_views call of three views (ray depth, depth statistics, absgrad, antialiasing, camera gradients)
    against render64 per view: shared leaves summed over the views, means2D, absgrad and the cameras per view."""
    lv, cam0, W, H, D = _row_scene("shell", 5, sh=True)
    cams = [cam0] + [synth.make_camera(k, W, H) for k in (3, 6)]
    mode = dict(aa=True, rd=True, ds=True, abs=True)
    views = []
    for v, cam in enumerate(cams):
        sc = Scene(lv, cam, W, H, D)
        st, clamped = _state(sc, True, True)
        cots, want, amb, _ = _truth(sc, mode, st, clamped, seed=1 + v)
        assert amb < 0.05, (v, amb)
        views.append((sc, cots, want))
    sc = views[0][0]
    for sname, s in SCALES:
        lvt, kw = _inputs(sc, GEOMETRY + APPEARANCE)
        camt = [{k: getattr(c, k).to(DEV).float().contiguous().requires_grad_(True)
                 for k in ("viewmatrix", "projmatrix", "campos")} for c in cams]
        settings = [_settings(sc, c["viewmatrix"], c["projmatrix"], c["campos"])._replace(bg=views[v][0].bg)
                    for v, c in enumerate(camt)]
        m2 = torch.zeros(len(cams), sc.P, 3, device=DEV, requires_grad=True)
        torch.use_deterministic_algorithms(det)
        try:
            out = R.rasterize_views(lvt["means3D"], m2, lvt["opacities"], settings=settings, antialiasing=True,
                                    ray_depth=True, depth_stats=True, absgrad=True, **kw)
            img = _image_dict(out, True)
            loss = sum((img[k][v] * c * s).sum() for v, (_, cots, _) in enumerate(views) for k, c in cots.items())
            wrt = {k: t for k, t in lvt.items() if t.requires_grad}
            gs = torch.autograd.grad(loss, list(wrt.values()) + [m2] + [c[k] for c in camt for k in c])
        finally:
            torch.use_deterministic_algorithms(False)
        fails = []
        shared = dict(zip(wrt, gs))
        total = {k: sum(w[k] for _, _, w in views) for k in list(shared) + ["opacities_mrow"]}
        _compare(shared, total, s, 1e-4, ("views", sname), fails)
        cg = gs[len(wrt) + 1:]
        for v, (_, _, want) in enumerate(views):
            got = {"means2D": gs[len(wrt)][v], "absgrad": m2.absgrad[v], "viewmatrix": cg[3 * v],
                   "projmatrix": cg[3 * v + 1], "campos": cg[3 * v + 2]}
            _compare(got, want, s, 1e-4, ("views", v, sname), fails)
        assert not fails, fails
