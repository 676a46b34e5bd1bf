"""The backward compositor's per-entry row sums on scenes built for their boundaries.

The compositor stages a block's contributors in batches of 32 from a queue of R3DG_QCAP, and sums each entry's row over
the block's pixels in sub-batches of 16 (8 from S = 18 on).  These scenes put stacks of 1, 15, 16, 17, 31, 32, 33, 255,
256 and 257 faint Gaussians on single pixel blocks, stacks on blocks cut by the image border (W, H not multiples of the
8x4 block), and wide Gaussians centred 50-500 px away from the blocks they composite in, on both sides and outside the
image.  Per row, |g - g64| <= TAU m_row against the fp64 truth (raster64.py, the bound of test_det_scale_gpu.py) at
mixed-sign unit and training-scale cotangents in both modes; in deterministic mode the gradients are bitwise equal
across two runs, the appearance-only backward's colour and feature rows bitwise the full backward's, and absgrad
changes no gradient."""
import math

import numpy as np
import pytest
import torch

import raster64
import test_camera_grad_gpu as cg
import test_raster_gpu as tr
from test_det_scale_gpu import TAU
from relightable3dgaussian_b200 import synth
from relightable3dgaussian_b200.rasterizer import rasterize_views

pytestmark = pytest.mark.gpu

W, H = 203, 150                                   # neither a multiple of 8 nor of 4: the last blocks are cut
COUNTS = (1, 15, 16, 17, 31, 32, 33, 255, 256, 257)
OUTPUTS = ("dL_dcolors", "dL_dfeatures", "dL_dopacity", "dL_dmeans2D", "dL_dcov3D")


def _scene(S, seed=0):
    """Inputs for run_ours (colors_precomp + cov3D_precomp, axis camera: depth is z)."""
    g = torch.Generator().manual_seed(seed)
    cam = synth.make_axis_camera(W, H)
    centres, sig, opac, z = [], [], [], []

    def add(n, u, v, s, o, depth):
        for _ in range(n):
            centres.append((u + 0.3 * float(torch.rand(1, generator=g)), v + 0.3 * float(torch.rand(1, generator=g))))
            sig.append(s); opac.append(o * (0.9 + 0.2 * float(torch.rand(1, generator=g))))
            z.append(depth + 0.5 * float(torch.rand(1, generator=g)))

    for i, n in enumerate(COUNTS):                # one stack per tile, 32 px apart: the stack's blocks see n entries
        add(n, 16 * (1 + 2 * (i % 6)) + 5.2, 16 * (1 + 2 * (i // 6)) + 2.1, 1.2, 0.015, 2.0)
    for n, u, v in ((17, W - 1.4, H - 0.7), (33, W - 2.2, 70.0), (31, 120.0, H - 1.1)):   # blocks cut by the border
        add(n, u, v, 1.2, 0.015, 2.0)
    far = ((-60, 40), (-250, 100), (W + 80, 20), (W + 300, 120), (90, -120), (40, H + 200), (150, -400), (100, 75))
    for k, (u, v) in enumerate(far):              # wide, centred 50-500 px away from most blocks they reach
        add(1, float(u), float(v), 40.0 + 20.0 * k, 0.35, 1.0 + 0.4 * k)
    P = len(z)
    z = torch.tensor(z)
    uv = torch.tensor(centres, dtype=torch.float64)
    x = ((uv[:, 0] + 0.5) * 2.0 / W - 1.0) * z.double() * cam.tanfovx
    y = ((uv[:, 1] + 0.5) * 2.0 / H - 1.0) * z.double() * cam.tanfovy
    means = torch.stack([x, y, z.double()], 1).float()
    sw = torch.tensor(sig, dtype=torch.float64) * z.double() * 2.0 * cam.tanfovx / W          # pixel sigma -> world
    c6 = torch.zeros(P, 6, dtype=torch.float64)
    c6[:, 0] = c6[:, 3] = c6[:, 5] = sw ** 2
    c6[:, 1] = 0.2 * sw ** 2                      # slightly anisotropic: the conic's off-diagonal term is exercised
    colors = torch.rand(P, 3, generator=g)
    feats = torch.rand(P, S, generator=g)
    kw = dict(means3D=means.numpy(), opacities=torch.tensor(opac)[:, None].float().numpy(),
              viewmatrix=cam.viewmatrix.numpy(), projmatrix=cam.projmatrix.numpy(), campos=cam.campos.numpy(),
              bg=np.array([0.0, 0.5, 1.0], np.float32), W=W, H=H, tan_fovx=cam.tanfovx, tan_fovy=cam.tanfovy,
              cx=cam.cx, cy=cam.cy, colors_precomp=colors.numpy(), cov3D_precomp=c6.float().numpy(),
              features=feats.numpy(), scale_modifier=1.0)
    return kw, cam


@pytest.mark.parametrize("S", [1, 5, 13, 16, 24])
def test_rows_match_fp64_truth(S):
    from relightable3dgaussian_b200 import _C_raster as C
    kw, _ = _scene(S)
    P = kw["means3D"].shape[0]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(False)
    try:
        o = tr.run_ours(C, **kw)
        mid = lambda n: o["mid"](n)                                                      # noqa: E731
        st = dict(point_list=mid("point_list"), ranges=mid("ranges"), n_contrib=mid("n_contrib"),
                  means2D=mid("means2D"), conic_opacity=mid("conic_opacity"), rgb=mid("rgb"), depths=mid("depths"),
                  features=torch.as_tensor(kw["features"]).cuda())
        nc = o["n_contrib"].reshape(H, W)
        assert int(nc.max()) >= max(COUNTS), "the deepest stack is not composited whole"
        walks = raster64.walks_of(st, W, H)
        amb = torch.zeros(H * W, dtype=torch.bool, device="cuda")
        rows = torch.zeros(P, dtype=torch.bool, device="cuda")
        for wk in walks:
            amb[wk.pix] = wk.ambiguous
            rows[wk.ids[wk.valid & (~wk.ambiguous)[:, None]]] = True
        assert float(amb.sum()) / (H * W) < 0.01
        live = (~amb).float().view(1, H, W)
        jac = raster64.cov3d_jacobian(torch.as_tensor(kw["means3D"]).cuda(), torch.as_tensor(kw["cov3D_precomp"]).cuda(),
                                      torch.as_tensor(kw["viewmatrix"]).cuda(), W, H, kw["tan_fovx"], kw["tan_fovy"])
        gu = torch.Generator().manual_seed(S)
        unit = [torch.randn(c, H, W, generator=gu).cuda() for c in (3, 1, 1, S)]
        sets = {"unit": unit, "training-scale": [c * 2.0 ** -21 for c in unit]}
        failures = {}
        for sname, cots in sets.items():
            cots = [c * live for c in cots]
            truth = raster64.row_truth(st, walks, cots, torch.as_tensor(kw["bg"]).cuda(), W, H, S, jac)
            for mode in (False, True):
                torch.use_deterministic_algorithms(mode)
                g = tr.run_ours(C, cots=cots, **kw)["grads"]
                nfail, worst = 0, 0.0
                for name in OUTPUTS:
                    g64, m = truth[name]
                    ours = g[name].reshape(P, -1)[:, :g64.shape[1]].double()
                    r = ((ours - g64).abs() / m.clamp_min(1e-300))[rows]
                    r = torch.where((m[rows] == 0) & (ours[rows] == 0), torch.zeros_like(r), r)
                    nfail += int((r > TAU).any(1).sum())
                    worst = max(worst, float(r.max()) if r.numel() else 0.0)
                print(f"[rows] S={S} {'det' if mode else 'default'} {sname}: worst |g - g64| / m_row {worst:.3e}")
                failures[(mode, sname)] = nfail
                if mode:
                    g2 = tr.run_ours(C, cots=cots, **kw)["grads"]
                    for name in OUTPUTS:
                        assert torch.equal(g[name], g2[name]), f"S={S} {sname} {name}: deterministic rerun differs"
    finally:
        torch.use_deterministic_algorithms(prev)
    assert not any(failures.values()), failures


def _views_grads(kw, cam, cots, *, appearance=False, absgrad=False):
    d = lambda a: torch.as_tensor(a).cuda().contiguous()                                 # noqa: E731
    leaves = dict(means3D=d(kw["means3D"]), opacities=d(kw["opacities"]), colors_precomp=d(kw["colors_precomp"]),
                  cov3D_precomp=d(kw["cov3D_precomp"]), features=d(kw["features"]))
    grad_of = ("colors_precomp", "features") if appearance else tuple(leaves)
    for k in grad_of:
        leaves[k].requires_grad_(True)
    camt = cg.camera_tensors(cam, grad=False)
    rs = cg.settings_of(cam, *camt, bg=d(kw["bg"]))
    m2d = torch.zeros(1, leaves["means3D"].shape[0], 3, device="cuda", requires_grad=not appearance)
    out = rasterize_views(leaves["means3D"], m2d, leaves["opacities"], settings=[rs], absgrad=absgrad,
                          **{k: v for k, v in leaves.items() if k not in ("means3D", "opacities")})
    names = list(grad_of) + ([] if appearance else ["means2D"])
    inputs = [leaves[k] for k in grad_of] + ([] if appearance else [m2d])
    gs = torch.autograd.grad([out[i] for i in range(2, 6)], inputs, grad_outputs=cots, allow_unused=True)
    res = dict(zip(names, gs))
    if absgrad:
        res["absgrad"] = m2d.absgrad.clone()
    return res


@pytest.mark.parametrize("S", [5, 24])
def test_deterministic_appearance_and_absgrad_rows(S):
    kw, cam = _scene(S, seed=1)
    g = torch.Generator().manual_seed(7)
    cots = [torch.randn(1, c, H, W, generator=g).cuda() for c in (3, 1, 1, S)]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        full = _views_grads(kw, cam, cots)
        app = _views_grads(kw, cam, cots, appearance=True)
        ab = _views_grads(kw, cam, cots, absgrad=True)
        ab2 = _views_grads(kw, cam, cots, absgrad=True)
    finally:
        torch.use_deterministic_algorithms(prev)
    for k in ("colors_precomp", "features"):
        assert torch.equal(app[k], full[k]), f"appearance-only {k} rows differ from the full backward's"
    for k, t in full.items():
        assert torch.equal(ab[k], t), f"absgrad changed {k}"
    assert torch.equal(ab["absgrad"], ab2["absgrad"])
    signed = full["means2D"][0, :, :2].abs()
    assert bool((ab["absgrad"] >= signed * (1 - 1e-4) - 1e-30).all())
    assert float(ab["absgrad"].max()) > 0 and not math.isnan(float(ab["absgrad"].sum()))
