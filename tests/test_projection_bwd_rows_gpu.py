"""The projection backward's leaf gradients (csrc/projection_bwd.cu) row by row against an fp64 truth.

For every Gaussian some unambiguous pixel composited, and every leaf output (dL_dmeans3D, dL_dscales, dL_drotations,
dL_dsh, dL_dopacity and dL_dcov3D), |g - g64| <= TAU_PROJ m_row, with g64 and m_row from proj64.leaf_truth on the
record gradients of raster64.row_truth.  The machinery is that of test_det_scale_gpu.py: the compositor's ambiguous
pixels get zero cotangents; the cotangent sets are unit and a training loss's on every scene in the plain mode (and
that times 2^-10 on shell-20k), unit in the other variants; both modes every time.  The projection's own
ambiguous rows (proj64.ambiguous_rows: the frustum clamp, the SH colour clamp, the antialiasing floor, 2D
conditioning) are excluded and counted.

Scenes built here, each asserting the path it is named for: frustum-edge (rows clamped in x, in y and in both),
sh-clamp (all 8 clamp patterns), near-and-axis (z in (0.2, 0.5], view directions on and near the optical axis),
quat-scale (non-unit quaternions with zero components, scale_modifier 0.37 / 2.5, scales 1e-4-1), and the existing
shell-20k, needles, inside-x0.6, inside-x1.8 and thresholds.  On shell, the SH layouts (D, M) and P = 128 k + 37 with
runs of 128 Gaussians behind the camera (CTAs with all, some and no rows live), and an M = 16 `shs` 4 bytes past a
16-byte boundary (the transposed slab).  On shell, frustum-edge and sh-clamp also antialiasing, the 3D filter, both,
three views in one call and the appearance-only backward; with camera gradients and absgrad switched on so that
every projection_bwd_kernel<DET, CAM, ABS, F3D> instantiation runs."""
import math

import numpy as np
import pytest
import torch

import proj64
import raster64
from helpers import case_inputs, edge_case
from relightable3dgaussian_b200 import synth

pytestmark = pytest.mark.gpu

# The worst |g - g64| / m_row in the default mode at unit cotangents over the scenes and variants below, measured on
# an NVIDIA H100 80GB HBM3 at a 700 W power limit: 9.4e-4, needles' dL_dsh, whose error is that of the compositor's
# colour row (its T recovered by division through alphas near the 0.99 clamp), which the per-term magnitudes of
# raster64 do not count.  The other scenes: at most 4.5e-4 (shell-D1-M16, dL_dopacity, again the compositor's row),
# most below 6e-5.  The compositor's TAU (test_det_scale_gpu.py, 2e-4) does not hold for them: one bound here, with
# the 4x of that file's convention.
TAU_PROJ_MEASURED = 9.4e-4
TAU_PROJ = 4 * TAU_PROJ_MEASURED
# needles: 5.3 % of its composited rows excluded on the H100 above (2D conditioning over 1e4), every other scene < 1 %
NEEDLES_EXCLUDED_MAX = 0.06
LEAF_OUT = {"means3D": "dL_dmeans3D", "scales": "dL_dscales", "rotations": "dL_drotations", "shs": "dL_dsh",
            "opacities": "dL_dopacity", "cov3D": "dL_dcov3D"}
GRADS = ["dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dfeatures", "dL_dcov3D", "dL_dsh",
         "dL_dscales", "dL_drotations"]
WORST = {}                       # (scene, variant, mode, cotangents) -> worst ratio, printed by the last test


def _axis_kw(means, scales, rots, shs, opac, W, H, cam, feats=None, mod=1.0):
    return dict(means3D=means.float(), opacities=opac.float(), scales=scales.float(), rotations=rots.float(),
                shs=shs.float(), features=feats, viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix,
                campos=cam.campos, bg=torch.tensor([0.0, 0.5, 1.0]), W=W, H=H, tan_fovx=cam.tanfovx,
                tan_fovy=cam.tanfovy, cx=cam.cx, cy=cam.cy, scale_modifier=mod, D=3)


def _random_rot(P, g):
    q = torch.randn(P, 4, generator=g)
    return q / q.norm(dim=1, keepdim=True)


def _frustum_edge():
    W, H = 160, 120
    g = torch.Generator().manual_seed(11)
    cam = synth.make_axis_camera(W, H)
    P = 6000
    z = 1.0 + 2.0 * torch.rand(P, generator=g)
    side = torch.randint(0, 8, (P,), generator=g)            # +-x, +-y and the four corners
    sx = torch.tensor([1, -1, 0, 0, 1, 1, -1, -1])[side].float()
    sy = torch.tensor([0, 0, 1, -1, 1, -1, 1, -1])[side].float()
    r = 1.0 + torch.rand(P, generator=g)                      # 1.0-2.0 x tan fov
    off = (torch.rand(P, 2, generator=g) * 2 - 1) * 0.9
    rx = torch.where(sx != 0, sx * r, off[:, 0]) * cam.tanfovx
    ry = torch.where(sy != 0, sy * r, off[:, 1]) * cam.tanfovy
    means = torch.stack([rx * z, ry * z, z], 1)
    # pixel sigma about half the centre's distance outside the image: the 2-sigma tails reach it
    fx = W / (2.0 * cam.tanfovx)
    sig_px = (((r - 1.0) * W / 2 + 4.0) / 2)[:, None] * (0.8 + 0.4 * torch.rand(P, 3, generator=g))
    scales = sig_px * z[:, None] / fx
    shs = torch.randn(P, 16, 3, generator=g) * 0.3
    return _axis_kw(means, scales, _random_rot(P, g), shs, 0.03 + 0.12 * torch.rand(P, 1, generator=g), W, H, cam)


def _sh_clamp():
    W, H = 160, 120
    g = torch.Generator().manual_seed(12)
    cam = synth.make_axis_camera(W, H)
    P = 8000
    z = 1.5 + 3.0 * torch.rand(P, generator=g)
    u = (torch.rand(P, 2, generator=g) * 2 - 1) * 0.95
    means = torch.stack([u[:, 0] * cam.tanfovx * z, u[:, 1] * cam.tanfovy * z, z], 1)
    scales = torch.exp(torch.rand(P, 3, generator=g) * 1.5 - 5.0) * z[:, None]
    shs = torch.randn(P, 16, 3, generator=g) * 0.5            # degree-3 rest terms large enough to matter
    pat = torch.arange(P) % 8
    neg = torch.stack([(pat >> c) & 1 for c in range(3)], 1).bool()
    shs[:, 0] = torch.where(neg, -3.5, 1.5) / proj64.SH_C0 * (0.6 + 0.8 * torch.rand(P, 3, generator=g))
    return _axis_kw(means, scales, _random_rot(P, g), shs, 0.1 + 0.3 * torch.rand(P, 1, generator=g), W, H, cam)


def _near_and_axis():
    W, H = 161, 121
    g = torch.Generator().manual_seed(13)
    cam = synth.make_axis_camera(W, H)
    P = 4000
    z = 0.2 + 0.3 * (1.0 - torch.rand(P, generator=g))        # (0.2, 0.5]
    ang = torch.where(torch.rand(P, generator=g) < 0.5, torch.zeros(P), torch.rand(P, generator=g) * 1e-3)
    phi = torch.rand(P, generator=g) * 2 * math.pi
    far = torch.rand(P, generator=g) < 0.4                    # the rest anywhere in view
    u = (torch.rand(P, 2, generator=g) * 2 - 1) * 0.9
    tx = torch.where(far, u[:, 0] * cam.tanfovx, torch.tan(ang) * torch.cos(phi))
    ty = torch.where(far, u[:, 1] * cam.tanfovy, torch.tan(ang) * torch.sin(phi))
    means = torch.stack([tx * z, ty * z, z], 1)
    scales = torch.exp(torch.rand(P, 3, generator=g) * 2.0 - 6.5) * z[:, None] * 4
    shs = torch.randn(P, 16, 3, generator=g) * 0.3
    return _axis_kw(means, scales, _random_rot(P, g), shs, 0.05 + 0.3 * torch.rand(P, 1, generator=g), W, H, cam)


def _quat_scale(mod):
    W, H = 160, 120
    g = torch.Generator().manual_seed(14)
    cam = synth.make_axis_camera(W, H)
    P = 6000
    size = torch.exp(torch.rand(P, 1, generator=g) * math.log(1e4) - math.log(1e4))      # 1e-4-1
    # the larger, the farther and fainter: the small ones are composited before the large ones saturate a pixel
    lvl = (size[:, 0].log10() + 4.0) / 4.0
    z = 1.0 + 3.0 * lvl + 0.3 * torch.rand(P, generator=g)
    u = (torch.rand(P, 2, generator=g) * 2 - 1) * 0.95
    means = torch.stack([u[:, 0] * cam.tanfovx * z, u[:, 1] * cam.tanfovy * z, z], 1)
    opac = torch.where(lvl > 0.6, 0.01 + 0.02 * torch.rand(P, generator=g), 0.05 + 0.5 * torch.rand(P, generator=g))
    scales = size * torch.exp(torch.rand(P, 3, generator=g) * 2.0 - 1.0) / mod
    q = _random_rot(P, g) * torch.exp(torch.rand(P, 1, generator=g) * math.log(16.0) - math.log(4.0))
    q[torch.rand(P, 4, generator=g) < 0.2] = 0.0
    q[(q == 0).all(1), 0] = 0.5
    shs = torch.randn(P, 16, 3, generator=g) * 0.3
    return _axis_kw(means, scales, q, shs, opac[:, None], W, H, cam, mod=mod)


def _edge(name):
    kw = edge_case(name)[0]
    kw = {k: (torch.as_tensor(v) if isinstance(v, np.ndarray) else v) for k, v in kw.items()}
    kw["D"] = 3
    return kw


def _shell(P=20_000, D=3, M=16):
    sc, cam = case_inputs(P, 160, 120, 5, view=1)
    shs = torch.zeros(P, M, 3)
    k = min(M, 16)
    shs[:, :k] = sc.shs[:, :k]
    return dict(means3D=sc.means3D, opacities=sc.opacities, scales=sc.scales, rotations=sc.rotations, shs=shs,
                features=sc.features, viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix, campos=cam.campos,
                bg=torch.tensor([0.0, 0.5, 1.0]), W=160, H=120, tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy, cx=cam.cx,
                cy=cam.cy, scale_modifier=1.0, D=D)


def _shell_ragged():
    """P = 128 k + 37 with runs of 128 Gaussians behind the camera: CTAs with all, some and no rows live."""
    kw = _shell(P=128 * 120 + 37)
    m = kw["means3D"].clone()
    cam = kw["viewmatrix"].double()
    behind = torch.zeros(m.shape[0], dtype=torch.bool)
    for b in range(0, 120, 3):
        behind[128 * b:128 * (b + 1)] = True                   # whole CTAs
    behind[128 * 7 + 5:128 * 7 + 70] = True                    # part of one
    fwd = torch.linalg.inv(cam[:3, :3])[2]                      # world direction of view z
    m[behind] = (m[behind].double() - 20.0 * fwd).float()       # 20 units behind: culled
    kw["means3D"] = m
    return kw


SCENES = {
    "shell-20k": _shell, "frustum-edge": _frustum_edge, "sh-clamp": _sh_clamp, "near-and-axis": _near_and_axis,
    "quat-scale-0.37": lambda: _quat_scale(0.37), "quat-scale-2.5": lambda: _quat_scale(2.5),
    "needles": lambda: _edge("needles"), "inside-x0.6": lambda: _edge("inside-x0.6"),
    "inside-x1.8": lambda: _edge("inside-x1.8"), "thresholds": lambda: _edge("thresholds"),
    "shell-D0-M1": lambda: _shell(D=0, M=1), "shell-D1-M4": lambda: _shell(D=1, M=4),
    "shell-D2-M9": lambda: _shell(D=2, M=9), "shell-D1-M16": lambda: _shell(D=1, M=16),
    "shell-ragged": _shell_ragged, "shell-shs-offset4": _shell,
}
# variant: (antialiasing, 3D filter, camera gradients, absgrad).  Plain runs on every scene; the others on the three
# scenes named in the module notes.  Between them every (CAM, ABS, F3D) combination runs, in both modes (DET).
VARIANTS = {"plain": (False, False, False, False), "plain-cam": (False, False, True, False),
            "plain-abs": (False, False, False, True), "aa": (True, False, True, True), "f3d": (False, True, False, False),
            "f3d-cam": (False, True, True, False), "f3d-abs": (False, True, False, True),
            "aa-f3d": (True, True, True, True)}
RICH = ("shell-20k", "frustum-edge", "sh-clamp")
CASES = [(s, "plain") for s in SCENES] + [(s, v) for s in RICH for v in VARIANTS if v != "plain"]


def _dev(kw, offset_shs=False):
    d = {}
    for k in ("means3D", "opacities", "scales", "rotations", "shs", "viewmatrix", "projmatrix", "campos", "bg"):
        d[k] = torch.as_tensor(kw[k]).float().cuda().contiguous()
    if offset_shs:                                             # data pointer 4 bytes past a 16-byte boundary
        buf = torch.zeros(d["shs"].numel() + 4, device="cuda")
        view = buf[1:1 + d["shs"].numel()].view(d["shs"].shape)
        view.copy_(d["shs"])
        assert view.data_ptr() % 16 == 4 and view.is_contiguous()
        d["shs"] = view
    f = kw.get("features")
    P = d["means3D"].shape[0]
    d["features"] = torch.as_tensor(f).float().cuda().contiguous() if f is not None else torch.empty(P, 0, device="cuda")
    return d


def _filter_3d(d):
    """f > 0 on most rows, 0 on some (every third row)."""
    P = d["means3D"].shape[0]
    g = torch.Generator().manual_seed(3)
    f = (0.002 + 0.01 * torch.rand(P, generator=g)).cuda()
    f[::3] = 0.0
    return f.contiguous()


def _forward(C, d, kw, aa, f3d):
    W, H, D = kw["W"], kw["H"], kw["D"]
    e = torch.empty(0, device="cuda")
    out = C.rasterize_gaussians(d["bg"], d["means3D"], d["features"], e, d["opacities"], d["scales"], d["rotations"],
                                kw["scale_modifier"], e, d["viewmatrix"], d["projmatrix"], kw["tan_fovx"],
                                kw["tan_fovy"], kw["cx"], kw["cy"], H, W, d["shs"], D, d["campos"], False, False, False,
                                antialiasing=aa, filter_3d=f3d)
    names = ["num_rendered", "n_contrib", "color", "opacity", "depth", "feature", "normal", "surface_xyz", "weights",
             "radii", "geom", "binning", "img"]
    o = dict(zip(names, out))
    P, S = d["means3D"].shape[0], d["features"].shape[1]
    o["mid"] = lambda n: C.debug_intermediate(n, P, S, W, H, o["geom"], o["img"], o["binning"], o["num_rendered"])
    return o


def _backward(C, d, kw, o, cots, aa, f3d, cam, ab, geometry=True):
    e = torch.empty(0, device="cuda")
    g = C.rasterize_gaussians_backward(d["bg"], d["means3D"], d["features"], o["radii"], e, d["scales"],
                                       d["rotations"], kw["scale_modifier"], e, d["viewmatrix"], d["projmatrix"],
                                       kw["tan_fovx"], kw["tan_fovy"], *cots, d["shs"], kw["D"], d["campos"], o["geom"],
                                       o["num_rendered"], o["binning"], o["img"], True, False, cam_grads=cam,
                                       geometry=geometry, antialiasing=aa, absgrad=ab, filter_3d=f3d,
                                       opacities=d["opacities"] if f3d is not None else None)
    torch.cuda.synchronize()
    return dict(zip(GRADS, g[:9]))


def _training_cots(o, S, W, H):
    """Cotangents of L1(color, gt) + 0.2 (1 - ssim(color, gt)) + L1 on up to three feature channels."""
    from relightable3dgaussian_b200 import losses
    g = torch.Generator(device="cuda").manual_seed(5)
    gt = torch.rand(3, H, W, device="cuda", generator=g)
    col = o["color"].detach().clone().requires_grad_(True)
    feat = o["feature"].detach().clone().requires_grad_(True)
    loss = (col - gt).abs().mean() + 0.2 * (1.0 - losses.ssim(col, gt))
    if S:
        gf = torch.rand(min(3, S), H, W, device="cuda", generator=g)
        loss = loss + (feat[:min(3, S)] - gf).abs().mean()
    dc, df = torch.autograd.grad(loss, [col, feat], allow_unused=True)
    df = torch.zeros_like(feat) if df is None else df
    z = torch.zeros(1, H, W, device="cuda")
    return [dc, z, z.clone(), df]


class View:
    """One forward's compositor state, its unambiguous rows and the projection's own ambiguous rows."""

    def __init__(self, C, d, kw, aa, f3d):
        W, H = kw["W"], kw["H"]
        self.o = o = _forward(C, d, kw, aa, f3d)
        mid = o["mid"]
        S = d["features"].shape[1]
        self.st = dict(point_list=mid("point_list"), ranges=mid("ranges"), n_contrib=mid("n_contrib"),
                       means2D=mid("means2D"), conic_opacity=mid("conic_opacity"), rgb=mid("rgb"), depths=mid("depths"),
                       features=d["features"])
        self.walks = raster64.walks_of(self.st, W, H)
        P = d["means3D"].shape[0]
        amb = torch.zeros(H * W, dtype=torch.bool, device="cuda")
        rows = torch.zeros(P, dtype=torch.bool, device="cuda")
        for wk in self.walks:
            amb[wk.pix] = wk.ambiguous
            rows[wk.ids[wk.valid & (~wk.ambiguous)[:, None]]] = True
        self.pix_amb = float(amb.float().mean())
        self.live = (~amb).float().view(1, H, W)
        self.clamped = mid("clamped").double()
        self.cam64 = proj64.Camera(d["viewmatrix"], d["projmatrix"], d["campos"], W, H, kw["tan_fovx"],
                                   kw["tan_fovy"], kw["scale_modifier"]).to("cuda")
        self.const = dict(clamped=self.clamped)
        if f3d is not None:
            self.const["filter_3d"] = f3d.double()
        leaves = self.leaves(d)
        crit = proj64.ambiguous_rows(leaves, self.const, self.cam64, kw["D"], aa=aa, f3d=f3d is not None)
        self.crit = {k: int((v & rows).sum()) for k, v in crit.items()}
        self.proj_amb = torch.stack(list(crit.values())).any(0)
        self.rows = rows & ~self.proj_amb
        self.n_rows = int(rows.sum())
        self.excluded = int((rows & self.proj_amb).sum()) / max(self.n_rows, 1)
        self.S = S

    @staticmethod
    def leaves(d):
        return dict(means3D=d["means3D"], opacities=d["opacities"], scales=d["scales"], rotations=d["rotations"],
                    shs=d["shs"])

    def cot_sets(self, W, H, seed):
        gu = torch.Generator().manual_seed(seed)
        unit = [torch.randn(c, H, W, generator=gu).cuda() for c in (3, 1, 1, self.S)]
        train = _training_cots(self.o, self.S, W, H)
        sets = {"unit": unit, "training": train, "training*2^-10": [c * 2.0 ** -10 for c in train]}
        return {k: [c * self.live for c in cs] for k, cs in sets.items()}

    def truth(self, d, kw, cots, aa, f3d):
        """{leaf: (g64, m_row)} on self.rows only (zeros elsewhere)."""
        W, H = kw["W"], kw["H"]
        rt = raster64.row_truth(self.st, self.walks, cots, d["bg"], W, H, self.S)
        g_rec, m_rec = proj64.rec_grad_from_rows(rt)
        idx = torch.nonzero(self.rows)[:, 0]
        sub = lambda t: t[idx]                                                            # noqa: E731
        lv = {k: sub(v) for k, v in self.leaves(d).items()}
        cs = {k: sub(v) for k, v in self.const.items()}
        out = proj64.leaf_truth(lv, cs, self.cam64, kw["D"], sub(g_rec), sub(m_rec), aa=aa, f3d=f3d is not None)
        # dL_dcov3D of the scales / rotations path: the gradient of the covariance the chain forms (s' when filtered)
        # (with the filter: at s' and the filtered opacity o coef, which the antialiasing term of the conic scales with)
        s, o = lv["scales"].double(), lv["opacities"].double()
        if f3d is not None:
            s, o, _ = proj64.filter3d_oracle.dilate(s, o, cs["filter_3d"])
        Sg = proj64.aa_oracle.cov3d_of(s * kw["scale_modifier"], lv["rotations"].double())
        cov = torch.stack([Sg[:, 0, 0], Sg[:, 0, 1], Sg[:, 0, 2], Sg[:, 1, 1], Sg[:, 1, 2], Sg[:, 2, 2]], 1)
        lc = dict(means3D=lv["means3D"], opacities=o.reshape(-1, 1), cov3D=cov, shs=lv["shs"])
        oc = proj64.leaf_truth(lc, cs, self.cam64, kw["D"], sub(g_rec), sub(m_rec), aa=aa, f3d=False)
        out["cov3D"] = oc["cov3D"]
        return idx, out


def _ratios(grads, idx, truth, names):
    """{leaf: worst ratio}, and the number of (row, leaf) pairs over TAU_PROJ."""
    worst, nfail = {}, 0
    for leaf in names:
        g64, m = truth[leaf]
        ours = grads[LEAF_OUT[leaf]].reshape(grads[LEAF_OUT[leaf]].shape[0], -1)[idx].double()[:, :g64.shape[1]]
        r = (ours - g64).abs() / m.clamp_min(1e-300)
        r = torch.where((m == 0) & (ours == 0), torch.zeros_like(r), r)
        worst[leaf] = float(r.max()) if r.numel() else 0.0
        nfail += int((r > TAU_PROJ).any(1).sum())
    return worst, nfail


@pytest.mark.parametrize("scene,variant", CASES, ids=[f"{s}-{v}" for s, v in CASES])
def test_projection_rows_match_fp64_truth(scene, variant):
    from relightable3dgaussian_b200 import _C_raster as C
    aa, use_f3d, cam, ab = VARIANTS[variant]
    kw = SCENES[scene]()
    d = _dev(kw, offset_shs=scene == "shell-shs-offset4")
    f3d = _filter_3d(d) if use_f3d else None
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        v = View(C, d, kw, aa, f3d)
        W, H = kw["W"], kw["H"]
        frac = v.excluded
        print(f"[proj-rows] {scene} {variant}: {int(v.rows.sum())} rows checked of {v.n_rows} composited by "
              f"unambiguous pixels; excluded {v.crit} ({100 * frac:.3f} %); ambiguous pixels {100 * v.pix_amb:.3f} %")
        _coverage(scene, v, kw)
        sets = v.cot_sets(W, H, seed=len(scene))
        if scene not in ("shell-20k",) and variant == "plain":
            sets = {k: sets[k] for k in ("unit", "training")}
        elif variant != "plain":
            sets = {"unit": sets["unit"]}
        failures = {}
        for sname, cots in sets.items():
            idx, truth = v.truth(d, kw, cots, aa, f3d)
            for det in (False, True):
                torch.use_deterministic_algorithms(det)
                g = _backward(C, d, kw, v.o, cots, aa, f3d, cam, ab)
                worst, nfail = _ratios(g, idx, truth, ["means3D", "scales", "rotations", "shs", "opacities", "cov3D"])
                mode = "det" if det else "default"
                WORST[(scene, variant, mode, sname)] = max(worst.values())
                print(f"[proj-rows] {scene} {variant} {mode} {sname}: worst |g - g64| / m_row "
                      + " ".join(f"{k} {x:.2e}" for k, x in worst.items()) + f"; {nfail} over {TAU_PROJ:.1e}")
                failures[(mode, sname)] = nfail
                if variant == "plain" and scene in RICH and sname == "unit":
                    app = _backward(C, d, kw, v.o, cots, aa, f3d, False, False, geometry=False)
                    w2, n2 = _ratios(app, idx, truth, ["shs"])
                    print(f"[proj-rows] {scene} appearance-only {mode} {sname}: dL_dsh worst {w2['shs']:.2e}")
                    failures[(mode, sname, "appearance-only")] = n2
    finally:
        torch.use_deterministic_algorithms(prev)
    assert frac < (NEEDLES_EXCLUDED_MAX if scene == "needles" else 0.01), \
        f"{scene} {variant}: {100 * frac:.3f} % of the rows excluded {v.crit}"
    assert not any(failures.values()), failures


def _coverage(scene, v, kw):
    """The path each scene is named for, among the rows checked."""
    rows = v.rows
    if scene == "frustum-edge":
        t = kw["means3D"].double().cuda() @ v.cam64.V[:3, :3] + v.cam64.V[3, :3]
        cx = (t[:, 0] / t[:, 2]).abs() > 1.3 * kw["tan_fovx"]
        cy = (t[:, 1] / t[:, 2]).abs() > 1.3 * kw["tan_fovy"]
        n = [int((rows & cx & ~cy).sum()), int((rows & cy & ~cx).sum()), int((rows & cx & cy).sum())]
        print(f"[proj-rows] frustum-edge: rows clamped in x only / y only / both: {n}")
        assert min(n) >= 200, n
    elif scene == "sh-clamp":
        c = v.clamped.long()
        pats = torch.bincount((c[:, 0] + 2 * c[:, 1] + 4 * c[:, 2])[rows], minlength=8)
        print(f"[proj-rows] sh-clamp: rows per clamp pattern {pats.tolist()}")
        assert int(pats.min()) >= 100, pats.tolist()
    elif scene == "near-and-axis":
        m = kw["means3D"].double().cuda()
        near = rows & (m[:, 2] <= 0.5)
        axis = rows & (m[:, :2].norm(dim=1) <= 1e-3 * m[:, 2] * 1.01)
        print(f"[proj-rows] near-and-axis: near rows {int(near.sum())}, on / near the axis {int(axis.sum())}")
        assert int(near.sum()) >= 500 and int(axis.sum()) >= 100
    elif scene.startswith("quat-scale"):
        q = kw["rotations"].cuda()
        n = q.norm(dim=1)
        zero = rows & (q == 0).any(1)
        print(f"[proj-rows] {scene}: rows with a zero component {int(zero.sum())}, |q| {float(n[rows].min()):.2f}-"
              f"{float(n[rows].max()):.2f}")
        assert int(zero.sum()) >= 100 and float(n[rows].min()) < 0.5 and float(n[rows].max()) > 2.0
    elif scene == "shell-ragged":
        live = v.o["radii"] > 0
        P = live.numel()
        per = [int(live[b:b + 128].sum()) for b in range(0, P, 128)]
        kinds = (sum(p == 0 for p in per), sum(0 < p < min(128, P - 128 * i) for i, p in enumerate(per)),
                 sum(p == min(128, P - 128 * i) for i, p in enumerate(per)))
        print(f"[proj-rows] shell-ragged: CTAs with no / some / all rows visible {kinds}")
        assert P % 128 == 37 and min(kinds) >= 1


@pytest.mark.parametrize("scene", RICH)
def test_three_views_rows_match_fp64_truth(scene):
    """rasterize_views with three cameras: the fp32 left fold (`acc`) of the views' leaf gradients, and dL_dsh rebuilt
    from the views' rank-1 factors, against the sum of the views' truths (and the sum of their m_row)."""
    from relightable3dgaussian_b200 import _C_raster as C
    kw = SCENES[scene]()
    d = _dev(kw)
    W, H = kw["W"], kw["H"]
    base = synth.make_axis_camera(W, H) if scene != "shell-20k" else None
    cams = []
    for k in range(3):
        if base is None:
            c = synth.make_camera(1 + k, W, H) if k else None
            vm = torch.as_tensor(kw["viewmatrix"]).float() if c is None else c.viewmatrix
            pm = torch.as_tensor(kw["projmatrix"]).float() if c is None else c.projmatrix
            cp = torch.as_tensor(kw["campos"]).float() if c is None else c.campos
        else:                                                   # the axis camera moved a little
            shift = torch.tensor([0.03 * k, -0.02 * k, 0.0])
            vm = base.viewmatrix.clone()
            vm[3, :3] -= shift
            pm = (vm.double() @ torch.linalg.inv(base.viewmatrix.double()) @ base.projmatrix.double()).float()
            cp = base.campos + shift
        cams.append((vm, pm, cp))
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        views, g_sum, m_sum, rows, cot_all = [], None, None, None, []
        for k, (vm, pm, cp) in enumerate(cams):
            dk = dict(d, viewmatrix=vm.cuda().contiguous(), projmatrix=pm.cuda().contiguous(),
                      campos=cp.cuda().contiguous())
            v = View(C, dk, kw, False, None)
            cots = v.cot_sets(W, H, seed=k + 1)["unit"]
            idx, truth = v.truth(dk, kw, cots, False, None)
            P = d["means3D"].shape[0]
            if g_sum is None:
                g_sum = {l: torch.zeros(P, t[0].shape[1], dtype=torch.float64, device="cuda") for l, t in truth.items()}
                m_sum = {l: torch.zeros_like(g_sum[l]) for l in truth}
                rows = torch.zeros(P, dtype=torch.bool, device="cuda")
                excl = torch.zeros(P, dtype=torch.bool, device="cuda")
            for l, (g64, m) in truth.items():
                g_sum[l][idx] += g64
                m_sum[l][idx] += m
            rows |= v.rows
            excl |= v.proj_amb & (v.o["radii"] > 0)
            cot_all.append(cots)
            views.append(dk)
        keep = rows & ~excl                                      # no view excluded the row
        vms = torch.stack([x["viewmatrix"] for x in views])
        pms = torch.stack([x["projmatrix"] for x in views])
        cps = torch.stack([x["campos"] for x in views])
        bgs = d["bg"][None].expand(3, 3).contiguous()
        e = torch.empty(0, device="cuda")
        camt = [(kw["tan_fovx"], kw["tan_fovy"], kw["cx"], kw["cy"])] * 3
        stacked = [torch.stack([c[i] for c in cot_all]).contiguous() for i in range(4)]
        failures = {}
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            out = C.rasterize_views(bgs, d["means3D"], d["features"], e, d["opacities"], d["scales"], d["rotations"],
                                    kw["scale_modifier"], e, vms, pms, camt, H, W, d["shs"], kw["D"], cps, False, False)
            geom, binning, img = out[10], out[11], out[12]
            g = C.rasterize_views_backward(bgs, d["means3D"], d["features"], e, d["scales"], d["rotations"],
                                           kw["scale_modifier"], e, vms, pms, camt, *stacked, d["shs"], kw["D"], cps,
                                           geom, binning, img, True)
            torch.cuda.synchronize()
            grads = dict(zip(GRADS, g[:9]))
            idx = torch.nonzero(keep)[:, 0]
            truth = {l: (g_sum[l][idx], m_sum[l][idx]) for l in g_sum}
            worst, nfail = _ratios(grads, idx, truth, ["means3D", "scales", "rotations", "shs", "opacities", "cov3D"])
            mode = "det" if det else "default"
            WORST[(scene, "views3", mode, "unit")] = max(worst.values())
            print(f"[proj-rows] {scene} views3 {mode}: {int(keep.sum())} rows, worst "
                  + " ".join(f"{k} {x:.2e}" for k, x in worst.items()))
            failures[mode] = nfail
    finally:
        torch.use_deterministic_algorithms(prev)
    assert not any(failures.values()), failures


def test_misaligned_rotations_view_is_bitwise_the_aligned_call():
    """A contiguous `rotations` view one float past an aligned base reaches the library as an aligned copy: in
    deterministic mode its images and every gradient equal the aligned call's bit for bit."""
    from relightable3dgaussian_b200 import _C_raster as C
    kw = _shell(P=5000)
    d = _dev(kw)
    P = d["rotations"].shape[0]
    buf = torch.zeros(4 * P + 4, device="cuda")
    buf[1:1 + 4 * P].copy_(d["rotations"].reshape(-1))
    rot_odd = buf[1:1 + 4 * P].view(P, 4)
    assert rot_odd.is_contiguous() and rot_odd.data_ptr() % 16 == 4
    gu = torch.Generator().manual_seed(9)
    cots = [torch.randn(c, kw["H"], kw["W"], generator=gu).cuda() for c in (3, 1, 1, 5)]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        res = []
        for rot in (d["rotations"], rot_odd):
            dd = dict(d, rotations=rot)
            o = _forward(C, dd, kw, False, None)
            g = _backward(C, dd, kw, o, cots, False, None, False, False)
            res.append((o, g))
    finally:
        torch.use_deterministic_algorithms(prev)
    (oa, ga), (ob, gb) = res
    for n in ("color", "opacity", "depth", "feature", "radii"):
        assert torch.equal(oa[n], ob[n]), n
    for n in GRADS:
        assert torch.equal(ga[n], gb[n]), n
    assert torch.equal(rot_odd, d["rotations"])                # the caller's view is untouched


def test_zz_print_worst_ratio_per_case():
    """The worst ratio of every (scene, variant, mode, cotangent set) the tests above measured, and TAU_PROJ's
    measurement: the default mode at unit cotangents."""
    for k, w in sorted(WORST.items()):
        print(f"[proj-rows] worst {k}: {w:.3e}")
    unit = [w for (s, v, m, c), w in WORST.items() if m == "default" and c == "unit"]
    if unit:
        print(f"[proj-rows] TAU_PROJ measurement (default, unit, every scene and variant): {max(unit):.3e}; "
              f"TAU_PROJ = {TAU_PROJ:.1e}")
