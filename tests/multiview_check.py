"""Comparison of the fused multi-view consistency losses with the fp64 oracle (multiview_oracle.py), shared by the GPU
tests: the kernel and oracle calls, the whole-map check of test_multiview_gpu.py, and the per-pixel checks of
test_multiview_edges_gpu.py (losses and counts, every gradient element, exact zeros off the pixels the definition
touches)."""
import torch

import multiview_oracle as mo
from relightable3dgaussian_b200 import multiview
from relightable3dgaussian_b200 import rasterizer as R

DEV = torch.device("cuda")
TAU = 1.0
# of the largest |fp64| element of the element's own pixel in that map: dL/ddepth at a pixel sums the geometric and
# photometric chains and other pixels' taps, which can nearly cancel (measured up to 8.5e-3 of the element on an H100)
FLOOR = {"depth": 1e-2, "normal": 2e-3}
# and, for elements that are small by cancellation, of the largest |fp64| element of the view's map: only for
# dL/ddepth, which the 1 / kNormEps amplification of short normals does not reach
FLOOR_VIEW = {"depth": 1e-5, "normal": 0.0}
TINY = 2.0 ** -120      # below fp32's normal range a product such as w = exp(-phi) underflows
FLOOR_ILL = 5e-2        # the same at photo pixels whose NCC gradient is a near-cancellation (Truth.ill)


def _settings(cams, W, H):
    return [R.GaussianRasterizationSettings(H, W, c.tanfovx, c.tanfovy, c.cx, c.cy, torch.zeros(3, device=DEV), 1.0,
                                            c.viewmatrix.float().to(DEV), torch.eye(4, device=DEV), 0,
                                            torch.zeros(3, device=DEV), False, True, True, False) for c in cams]


def _kernel(depth, normal, gray, settings, pairs, cot, tau=TAU):
    """(geo, photo, counts, dL/ddepth, dL/dnormal) of the fused loss for the loss sum(geo * cot[0] + photo * cot[1]);
    a cotangent of None leaves that output out of the loss."""
    d, n = depth.detach().clone().requires_grad_(), normal.detach().clone().requires_grad_()
    view, cams, idx, tau = multiview._prepare(d, n, gray, settings, pairs, tau)
    geo, photo, counts = multiview._Consistency.apply(d, n, gray, view, cams, idx, tau)
    loss = sum((o * c).sum() for o, c in zip((geo, photo), cot) if c is not None)
    gd, gn = torch.autograd.grad(loss, [d, n])
    return geo.detach(), photo.detach(), counts, gd, gn


def _oracle(depth, normal, gray, cams, pairs, cot, counts, dtype, tau=TAU):
    d = depth.detach().to(dtype).requires_grad_()
    n = normal.detach().to(dtype).requires_grad_()
    geo, photo, info = mo.consistency(d, n, gray.to(dtype), cams, pairs, tau, counts=counts, info=True)
    loss = sum((o * c.to(dtype)).sum() for o, c in zip((geo, photo), cot) if c is not None)
    gd, gn = torch.autograd.grad(loss, [d, n], allow_unused=True) if torch.is_tensor(loss) else (None, None)
    gd = torch.zeros_like(d) if gd is None else gd
    gn = torch.zeros_like(n) if gn is None else gn
    return geo.detach(), photo.detach(), gd, gn, info


def _rel(a, b, keep):
    fin = lambda t: torch.isfinite(t).reshape(*keep.shape, -1).all(-1)
    keep = keep & fin(a) & fin(b)
    a, b = a.double()[keep], b.double()[keep]
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def check_against_oracle(depth, normal, gray, cams, pairs, seed=0, border_budget=1e-3):
    """Kernel vs fp64 oracle within max(1e-6, 4 e_ref) (+ the share of pixels on a decision boundary for the losses),
    e_ref the fp32 oracle's own error; gradient maps in relative L2 off the boundary pixels."""
    V, _, H, W = depth.shape
    settings = _settings(cams, W, H)
    g = torch.Generator(device=DEV).manual_seed(seed)
    B = len(pairs)
    cot = (torch.rand(B, device=DEV, generator=g) + 0.5, torch.rand(B, device=DEV, generator=g) + 0.5)
    kg, kp, counts, kgd, kgn = _kernel(depth, normal, gray, settings, pairs, cot)
    cl = counts.cpu().tolist()
    tg, tp, tgd, tgn, info = _oracle(depth, normal, gray, cams, pairs, cot, cl, torch.float64)
    fg, fp, fgd, fgn, _ = _oracle(depth, normal, gray, cams, pairs, cot, cl, torch.float32)
    keep_d = torch.ones(V, H * W, dtype=torch.bool, device=DEV)
    keep_n = torch.ones(V, H * W, dtype=torch.bool, device=DEV)
    for b, ((r, n), e) in enumerate(zip(pairs, info)):
        gb, pb = mo.borderline(e, TAU, W, H)
        if r != n:          # for (v, v) every edge pixel reprojects onto the image bound by construction
            assert int((gb | pb).sum()) <= border_budget * H * W, (b, int(gb.sum()), int(pb.sum()))
        allow_g = int(gb.sum()) * TAU / max(cl[b][0], 1)
        allow_p = int((gb | pb).sum()) * mo.MAX_COST / max(cl[b][1], 1)
        for k, t, f, allow in ((kg[b], tg[b], fg[b], allow_g), (kp[b], tp[b], fp[b], allow_p)):
            e_ref = abs(float(f) - float(t))
            assert abs(float(k) - float(t)) <= max(1e-6, 4 * e_ref) + allow, (b, float(k), float(t), e_ref, allow)
        bad = gb | pb
        keep_d[r] &= ~bad
        keep_n[r] &= ~bad
        q = e["q"][bad]
        x0, y0 = q[:, 0].floor().long().clamp(0, W - 1), q[:, 1].floor().long().clamp(0, H - 1)
        for dx in (0, 1):
            for dy in (0, 1):
                keep_d[n, (y0 + dy).clamp(max=H - 1) * W + (x0 + dx).clamp(max=W - 1)] = False
    kd, td, fd = kgd.reshape(V, -1), tgd.reshape(V, -1), fgd.reshape(V, -1)
    # where the fp32 formulation overflows (e.g. unbounded depths off a rendered silhouette) it has no error to compare
    keep_d &= torch.isfinite(fd)
    keep_n &= torch.isfinite(fgn.reshape(V, 3, -1)).all(1)
    rk, rf = _rel(kd, td, keep_d), _rel(fd, td, keep_d)
    assert rk <= max(1e-6, 4 * rf), ("depth", rk, rf)
    kn, tn, fn = (t.reshape(V, 3, -1).transpose(1, 2) for t in (kgn, tgn, fgn))
    rk, rf = _rel(kn, tn, keep_n), _rel(fn, tn, keep_n)
    assert rk <= max(1e-6, 4 * rf), ("normal", rk, rf)
    assert torch.isfinite(kgd).all() and torch.isfinite(kgn).all()
    return kg, kp, counts


# ---- per-pixel checks ---------------------------------------------------------------------------------------------


def _taps(q, W, H):
    """Flat indices [N,4] of the four bilinear taps of q [N,2] (clamped into the image; q may be NaN)."""
    q = torch.nan_to_num(q, nan=-2.0, posinf=-2.0, neginf=-2.0).clamp(-2.0, float(max(W, H) + 2))
    x0, y0 = q[:, 0].floor().long(), q[:, 1].floor().long()
    out = [(y0 + dy).clamp(0, H - 1) * W + (x0 + dx).clamp(0, W - 1) for dy in (0, 1) for dx in (0, 1)]
    return torch.stack(out, 1)


class Truth:
    """The fp64 and fp32 oracle of one call (losses, gradients, per-pair dicts), the masks of the elements the
    per-pixel checks skip (borderline pixels and their taps), and the masks of the elements the definition touches."""

    def __init__(self, depth, normal, gray, cams, pairs, cot, counts, tau=TAU):
        V, _, H, W = depth.shape
        self.V, self.H, self.W, self.pairs, self.tau = V, H, W, pairs, tau
        cl = counts.cpu().tolist()
        self.tg, self.tp, self.gd, self.gn, self.info = _oracle(depth, normal, gray, cams, pairs, cot, cl,
                                                                torch.float64, tau)
        self.fg, self.fp, self.fgd, self.fgn, _ = _oracle(depth, normal, gray, cams, pairs, cot, cl, torch.float32, tau)
        self.skip = torch.zeros(V, H * W, dtype=torch.bool, device=DEV)      # depth and normal elements not compared
        self.touch_d = torch.zeros(V, H * W, dtype=torch.bool, device=DEV)   # may be nonzero in dL/ddepth
        self.touch_n = torch.zeros(V, H * W, dtype=torch.bool, device=DEV)   # may be nonzero in dL/dnormal
        # low-contrast, weakly correlated patches (var a var b < 1e-6, c > 0.7): the NCC gradient is a difference of
        # nearly equal terms over sqrt(var a var b + 1e-8), so fp32 rounding of the warped grey values moves it by up
        # to a few percent of the pixel's own gradient (traced on the flat scene: every element beyond FLOOR lies at
        # such a pixel, 4e-3 to 4e-2 px from any texel edge)
        self.ill = torch.zeros(V, H * W, dtype=torch.bool, device=DEV)
        # D |n_c| / |d| at photo pixels: the homography divides by d, so its fp32 error, relative to the pixel's own
        # gradient, grows with it (near-perpendicular planes); the floor gains 1e-5 of it
        self.cond = torch.zeros(V, H * W, dtype=torch.float64, device=DEV)
        self.border, self.kinks = [], []
        for (r, n), e in zip(pairs, self.info):
            gb, pb = mo.borderline_edges(e, tau, W, H)
            self.border.append((int(gb.sum()), int((gb | pb).sum())))
            bad = gb | pb
            # and for the gradients only: a q or a warped tap within fp32 reach of a grid line, where the derivative
            # of the bilinear sample jumps (the definition's own kink; the pixel's validity does not change there)
            # phi within fp32 reach of 0: the direction of p' - p, and so the geo gradient, is set by rounding
            kink = (e["geo"] & ((e["q_grid"] < 1) | (e["phi"] < 1e-3))) \
                | (e["photo"] & (torch.nan_to_num(e["tap_grid"], nan=2.0) < 1))
            self.kinks.append(int(kink.sum()))
            self.skip[r] |= bad | kink
            self.skip[n, _taps(e["q_raw"][bad], W, H).reshape(-1)] = True
            self.touch_d[r] |= e["geo"] | bad
            self.touch_d[n, _taps(e["q_raw"][e["geo"] | bad], W, H).reshape(-1)] = True
            self.touch_n[r] |= e["photo"] | bad
            nc = (e["nlen"] / 1e-12).clamp(max=1.0)
            cond = torch.where(e["photo"], e["D"] * nc / e["d"], torch.zeros_like(e["D"])).double()
            self.cond[r] = torch.maximum(self.cond[r], torch.nan_to_num(cond, nan=0.0))
            self.ill[r] |= e["photo"] & (torch.nan_to_num(e["va"] * e["vb"], nan=1.0) < 1e-6) & (e["c"] > 0.7)


def check_losses(k, t, label=""):
    """Losses within max(1e-6, 4 e_ref) plus the borderline pixels' share, and counts equal to the oracle's up to the
    borderline pixels of each pair.  k = (geo, photo, counts)."""
    kg, kp, counts = k
    cl = counts.cpu().tolist()
    for b, e in enumerate(t.info):
        nb_g, nb_p = t.border[b]
        want = (int(e["geo"].sum()), int(e["photo"].sum()))
        assert abs(cl[b][0] - want[0]) <= nb_g and abs(cl[b][1] - want[1]) <= nb_p, (label, b, cl[b], want, t.border[b])
        allow_g = nb_g * min(t.tau, 1.0) / max(cl[b][0], 1)        # w phi = phi exp(-phi) < min(tau, 1 / e)
        allow_p = nb_p * mo.MAX_COST / max(cl[b][1], 1)
        for name, kk, tt, ff, allow in (("geo", kg[b], t.tg[b], t.fg[b], allow_g),
                                        ("photo", kp[b], t.tp[b], t.fp[b], allow_p)):
            e_ref = abs(float(ff) - float(tt))
            assert abs(float(kk) - float(tt)) <= max(1e-6, 4 * e_ref) + allow, \
                (label, name, b, float(kk), float(tt), e_ref, allow)


def det_resolution(cot, counts):
    """2^(e - 48), the fixed-point unit of a deterministic-mode term when the class exponent e is the cotangent's
    (the largest |dL/dgeo[b]| / max(n_geo, 1) and |dL/dphoto[b]| / max(n_photo, 1))."""
    cl = counts.cpu().tolist()
    m = max([abs(float(c[b])) / max(cl[b][k], 1) for k, c in enumerate(cot) if c is not None for b in range(len(cl))]
            + [0.0])
    return 2.0 ** (torch.tensor(m).log2().floor().item() - 48) if m > 0 else 0.0


def check_pixels(gd, gn, t, label="", unit=0.0):
    """Every gradient element off the borderline pixels and their taps within 8 |fp32 - fp64| + FLOOR[map] P of the fp64
    truth, P the largest |fp64| element of the same pixel in that map (the element itself for dL/ddepth, the three
    channels for dL/dnormal), so each pixel is held to its own scale, whatever the rest of its view holds; finite
    wherever the truth is; and exactly 0 wherever no valid pixel or tap of any pair lies.  In deterministic mode `unit`
    is det_resolution(): each of an element's terms is rounded to it (or to 2^-94 of the class's largest term when
    that raises the exponent), and 64 units are allowed.  Returns the worst element
    of each map as ((|kernel - fp64| - 8 |fp32 - fp64|) / P, the share of P the floor has to cover, view, index).""" 
    V, HW = t.V, t.H * t.W
    worst = {}
    for name, k, tr, f, touch in (("depth", gd.reshape(V, 1, HW), t.gd.reshape(V, 1, HW), t.fgd.reshape(V, 1, HW),
                                   t.touch_d), ("normal", gn.reshape(V, 3, HW), t.gn.reshape(V, 3, HW),
                                                t.fgn.reshape(V, 3, HW), t.touch_n)):
        assert bool(torch.isfinite(k[torch.isfinite(tr)]).all()), (label, name, "not finite where the truth is")
        stray = (k != 0) & ~touch[:, None, :]
        assert not bool(stray.any()), (label, name, "written off the pixels the definition touches",
                                       int(stray.sum()), stray.nonzero()[:4].tolist(), k[stray][:4].tolist())
        P = tr.abs().amax(dim=1, keepdim=True)
        coef = torch.where(t.ill[:, None, :], FLOOR_ILL, FLOOR[name]) + 1e-5 * t.cond[:, None, :]
        err = (k.double() - tr).abs()
        view = tr.abs().amax(dim=(1, 2), keepdim=True)
        res = max(unit, 2.0 ** (float(tr.abs().max().clamp_min(1e-300).log2().floor()) - 94)) if unit else 0.0
        bound = 8 * (f.double() - tr).abs() + coef * P + FLOOR_VIEW[name] * view + TINY + 64 * res
        keep = ~t.skip[:, None, :]
        over = keep & ~(err <= bound)
        rel = torch.where(keep & (P > 0), (err - 8 * (f.double() - tr).abs()).clamp_min(0) / P.clamp_min(1e-300),
                          torch.zeros_like(err))
        i = int(rel.argmax())
        worst[name] = (float(rel.reshape(-1)[i]), i // (rel.shape[1] * HW), i % HW)
        if bool(over.any()):
            j = over.nonzero()[0].tolist()
            raise AssertionError((label, name, "element outside its bound", int(over.sum()), j, float(k[tuple(j)]),
                                  float(tr[tuple(j)]), float(f[tuple(j)]), float(P[j[0], 0, j[2]])))
    return worst
