"""The fp64 truth of the projection backward (proj64.py) on the CPU: against the C oracle (oracle_preprocess_backward,
an fp32 mirror of the reference's preprocess backward) row by row, against central differences where the reference's
backward is a true derivative, and the frustum clamp's departure from it pinned explicitly.

Geometry built to reach every branch: view directions on both sides of the 1.3 tan(fov) clamp in x, in y and in both,
all 8 SH clamp patterns, non-unit quaternions (norms 0.25-4) with exactly-zero components, scale_modifier 0.37, 1 and
2.5, SH degrees 0-3 at M = 16, and the colors_precomp + cov3D_precomp path."""
import numpy as np
import pytest
import torch

import proj64
from oracle import oracle
from relightable3dgaussian_b200 import synth

# The worst |oracle - g64| / m_row over every case below, measured with the fp32 C oracle built by oracle/build.sh
# (x86-64 CPU): 2.6e-4, dL_dscales at D = 3, scale_modifier 2.5 (a 2D covariance near the 1e4 conditioning cut,
# whose fp32 determinant carries the error).  TAU_CPU leaves 4x, the convention of the GPU bounds.
TAU_CPU_MEASURED = 2.6e-4
TAU_CPU = 4 * TAU_CPU_MEASURED
W, H = 160, 120


def _scene(P, D, mod, seed, precomp=False):
    """Leaves (fp32 torch), clamp flags, camera and record gradients of P adversarial Gaussians (see the module notes)."""
    g = torch.Generator().manual_seed(seed)
    cam = synth.make_camera(1, W, H)
    V = cam.viewmatrix.double()
    Lx, Ly = 1.3 * cam.tanfovx, 1.3 * cam.tanfovy
    tz = 0.3 + 4.7 * torch.rand(P, generator=g, dtype=torch.float64)
    rx = (torch.rand(P, generator=g, dtype=torch.float64) * 2 - 1) * 2.0 * Lx       # half of them clamped in x
    ry = (torch.rand(P, generator=g, dtype=torch.float64) * 2 - 1) * 2.0 * Ly
    rx[:P // 8] = 0.0                                                                  # on the optical axis
    t = torch.stack([rx * tz, ry * tz, tz], 1)
    means = ((t - V[3, :3]) @ torch.linalg.inv(V[:3, :3])).float()
    # per-row size 1e-4-1 relative to depth, axis ratios up to ~30 (needles are the GPU scene `needles`)
    size = torch.exp(torch.rand(P, 1, generator=g) * np.log(1e4) - np.log(1e4))
    scales = size * torch.exp(torch.rand(P, 3, generator=g) * 3.4 - 1.7) * tz[:, None].float()
    q = torch.randn(P, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True) * torch.exp(torch.rand(P, 1, generator=g) * np.log(16.0) - np.log(4.0))
    q[torch.rand(P, 4, generator=g) < 0.15] = 0.0                                      # exactly-zero components
    q[(q == 0).all(1), 0] = 1.0
    sh = torch.randn(P, 16, 3, generator=g) * 0.4
    # DC so that the raw colour 0.5 + sum_k w_k sh_k lands on either side of 0: every clamp pattern (pattern = row % 8)
    sign = torch.tensor([[(k >> c) & 1 for c in range(3)] for k in range(8)], dtype=torch.float32)[torch.arange(P) % 8]
    sh[:, 0] = torch.where(sign > 0, -4.0, 2.0) / proj64.SH_C0 * (0.5 + torch.rand(P, 3, generator=g))
    leaves = dict(means3D=means, opacities=torch.rand(P, 1, generator=g))
    if precomp:
        C = proj64.aa_oracle.cov3d_of(scales.double(), q.double(), 1.0)
        leaves["cov3D"] = torch.stack([C[:, 0, 0], C[:, 0, 1], C[:, 0, 2], C[:, 1, 1], C[:, 1, 2], C[:, 2, 2]], 1).float()
        leaves["colors"] = torch.rand(P, 3, generator=g)
    else:
        leaves.update(scales=scales, rotations=q, shs=sh)
    cam64 = proj64.Camera(cam.viewmatrix, cam.projmatrix, cam.campos, W, H, cam.tanfovx, cam.tanfovy, mod)
    # the forward's clamp flags, decided in fp64 (rows where fp32 may decide otherwise are excluded)
    d = means.double() - cam64.campos
    d = d / d.norm(dim=1, keepdim=True)
    w = torch.func.vmap(lambda dd: proj64.sh_basis(D, dd))(d)[:, :, None] * sh.double()
    clamped = ((0.5 + w.sum(1)) < 0).to(torch.uint8)
    g_rec = torch.randn(P, 10, generator=g, dtype=torch.float64) * torch.exp(
        torch.randn(P, 1, generator=g, dtype=torch.float64))
    return leaves, clamped, cam, cam64, g_rec


def _oracle_grads(leaves, clamped, cam, D, mod, g_rec):
    """oracle_preprocess_backward on record gradients g_rec (REC order, conic b the true derivative)."""
    P = g_rec.shape[0]
    n = lambda t: np.ascontiguousarray(t.detach().numpy(), np.float32)                  # noqa: E731
    g = n(g_rec)
    dmean2 = np.ascontiguousarray(g[:, 0:3])
    dconic = np.ascontiguousarray(np.stack([g[:, 3], 0.5 * g[:, 4], np.zeros(P, np.float32), g[:, 5]], 1))
    dcol = np.ascontiguousarray(g[:, 7:10])
    if "cov3D" in leaves:
        cov = n(leaves["cov3D"])
    else:
        C = proj64.aa_oracle.cov3d_of(leaves["scales"].double(), leaves["rotations"].double(), mod)
        cov = n(torch.stack([C[:, 0, 0], C[:, 0, 1], C[:, 0, 2], C[:, 1, 1], C[:, 1, 2], C[:, 2, 2]], 1))
    M = 16 if "shs" in leaves else 0
    out = dict(dL_dmeans3D=np.zeros((P, 3), np.float32), dL_dcov3D=np.zeros((P, 6), np.float32),
               dL_dsh=np.zeros((P, max(M, 1), 3), np.float32), dL_dscales=np.zeros((P, 3), np.float32),
               dL_drotations=np.zeros((P, 4), np.float32))
    import ctypes
    p = oracle._p
    shs = n(leaves["shs"]) if M else None
    oracle.lib().oracle_preprocess_backward(
        ctypes.c_int(P), ctypes.c_int(D), ctypes.c_int(M), p(n(leaves["means3D"])), p(np.ones(P, np.int32)), p(shs),
        p(np.ascontiguousarray(clamped.numpy())), p(n(leaves["scales"]) if "scales" in leaves else None),
        p(n(leaves["rotations"]) if "rotations" in leaves else None), ctypes.c_float(mod), p(cov),
        p(n(cam.viewmatrix)), p(n(cam.projmatrix)), ctypes.c_int(W), ctypes.c_int(H), ctypes.c_float(cam.tanfovx),
        ctypes.c_float(cam.tanfovy), p(n(cam.campos)), p(dmean2), p(dconic), p(dcol), p(out["dL_dmeans3D"]),
        p(out["dL_dcov3D"]), p(out["dL_dsh"]), p(out["dL_dscales"]), p(out["dL_drotations"]))
    return out


CASES = [(D, mod) for D in range(4) for mod in (0.37, 1.0, 2.5)] + [("precomp", 1.0)]


@pytest.mark.parametrize("D,mod", CASES, ids=[f"D{d}-mod{m}" for d, m in CASES])
def test_truth_matches_c_oracle_row_by_row(D, mod):
    precomp = D == "precomp"
    D = 3 if precomp else D
    P = 3000
    leaves, clamped, cam, cam64, g_rec = _scene(P, D, mod, seed=D * 7 + int(mod * 100), precomp=precomp)
    crit = proj64.ambiguous_rows(leaves, dict(clamped=clamped), cam64, D)
    amb = torch.stack(list(crit.values())).any(0)
    assert float(amb.float().mean()) < 0.01, {k: int(v.sum()) for k, v in crit.items()}
    truth = proj64.leaf_truth(leaves, dict(clamped=clamped), cam64, D, g_rec, g_rec.abs())
    orc = _oracle_grads(leaves, clamped, cam, D, mod, g_rec)
    names = {"means3D": "dL_dmeans3D", "scales": "dL_dscales", "rotations": "dL_drotations", "shs": "dL_dsh",
             "cov3D": "dL_dcov3D"}
    t = torch.as_tensor(cam.viewmatrix).double()
    tt = leaves["means3D"].double() @ t[:3, :3] + t[3, :3]
    cx = (tt[:, 0] / tt[:, 2]).abs() > 1.3 * cam.tanfovx
    cy = (tt[:, 1] / tt[:, 2]).abs() > 1.3 * cam.tanfovy
    assert int((cx & ~cy).sum()) > 300 and int((cy & ~cx).sum()) > 300 and int((cx & cy).sum()) > 300
    if not precomp:
        pats = (clamped[:, 0] + 2 * clamped[:, 1] + 4 * clamped[:, 2]).long()
        assert torch.bincount(pats[~amb], minlength=8).min() >= 100
    worst = 0.0
    for leaf, key in names.items():
        if leaf not in truth:
            continue
        g64, m = truth[leaf]
        ours = torch.as_tensor(orc[key]).reshape(P, -1).double()[:, :g64.shape[1]]
        r = ((ours - g64).abs() / m.clamp_min(1e-300))[~amb]
        r = torch.where((m[~amb] == 0) & (ours[~amb] == 0), torch.zeros_like(r), r)
        w = float(r.max())
        print(f"[proj64-cpu] D={D} mod={mod} {leaf}: worst |oracle - g64| / m_row {w:.3e}")
        worst = max(worst, w)
        assert w <= TAU_CPU, (leaf, w)


def test_truth_is_central_differences_of_the_forward_where_unclamped():
    """On rows the frustum does not clamp (and at scale_modifier 1), record()'s Jacobian is the derivative of its
    values, which are the forward's: fp64 central differences agree."""
    P, D = 64, 3
    leaves, clamped, cam, cam64, _ = _scene(P, D, 1.0, seed=5)
    t = torch.as_tensor(cam.viewmatrix).double()
    tt = leaves["means3D"].double() @ t[:3, :3] + t[3, :3]
    keep = ((tt[:, 0] / tt[:, 2]).abs() < 1.2 * cam.tanfovx) & ((tt[:, 1] / tt[:, 2]).abs() < 1.2 * cam.tanfovy)
    assert int(keep.sum()) >= 10
    for i in torch.nonzero(keep)[:, 0].tolist()[:10]:
        lv = {k: v[i].double() for k, v in leaves.items()}
        cs = dict(clamped=clamped[i].double())
        J = torch.func.jacrev(lambda x: proj64.record(x, cs, cam64, D)[0])(lv)
        for k, x in lv.items():
            for j in range(x.numel()):
                h = 1e-6 * max(float(x.reshape(-1)[j].abs()), 1e-2 * float(x.abs().max()))
                e = torch.zeros_like(x).reshape(-1)
                e[j] = h
                e = e.view_as(x)
                f = lambda y: proj64.record(dict(lv, **{k: y}), cs, cam64, D)[0]          # noqa: E731
                cd = (f(x + e) - f(x - e)) / (2 * h)
                an = J[k].reshape(10, -1)[:, j]
                assert torch.allclose(an, cd, rtol=1e-5, atol=1e-5 * float(cd.abs().max()) + 1e-8), (k, j, an, cd)


def test_frustum_clamp_j02_term_is_twice_the_true_tz_derivative():
    """The reference's backward keeps 2 h_x t0 / tz^3 dL/dJ02 in dL/dtz of a clamped row, twice the derivative of
    J02 = -h_x clamp(tx / tz) tz / tz^2 = -h_x L / tz.  proj64 restates it (autograd with t0 detached); pin it."""
    hx, L = 200.0, 1.3 * 0.36
    tx, tz = torch.tensor(2.0 * L * 3.0, dtype=torch.float64), torch.tensor(3.0, dtype=torch.float64)
    assert float(tx / tz) > L
    ref = torch.func.grad(lambda z: -hx * proj64._clamp_t(tx, z, L) / (z * z))(tz)
    true = lambda z: -hx * (tx / z).clamp(-L, L) * z / (z * z)                           # noqa: E731
    h = 1e-6
    cd = (true(tz + h) - true(tz - h)) / (2 * h)
    assert abs(float(ref) / float(cd) - 2.0) < 1e-8, (float(ref), float(cd))
    assert float(torch.func.grad(lambda x: -hx * proj64._clamp_t(x, tz, L) / (tz * tz))(tx)) == 0.0
