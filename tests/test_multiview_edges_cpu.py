"""The adversarial multi-view scenes without a GPU: every scene takes the branches it exists for (the same coverage
the GPU tests assert, here on the fp64 oracle), and the oracle's gradients match central finite differences at pixels
of those branches (taps next to holes, normals shorter than F.normalize's eps, flat patches, planes near the camera
centre), with the weights and counts held fixed."""
import pytest
import torch

import multiview_edges as me
import multiview_oracle as mo

TAU = 1.0


def _maps(name):
    build, pairs, cov = me.SCENES[name]
    depth, normal, gray, cams = build()
    return depth.float().double(), normal.float().double(), gray.float().double(), cams, pairs, cov


@pytest.mark.parametrize("name", list(me.SCENES))
def test_scene_coverage(name):
    d, n, g, cams, pairs, cov = _maps(name)
    _, _, infos = mo.consistency(d, n, g, cams, pairs, TAU, info=True)
    for branch, (count, least) in cov(infos, (d, n, g, cams)).items():
        assert count >= least, (name, branch, count, least)


def _sample(mask, k, seed):
    idx = mask.nonzero().squeeze(1)
    assert idx.numel() > 0
    perm = torch.randperm(idx.numel(), generator=torch.Generator().manual_seed(seed))
    return idx[perm[:k]].tolist()


BRANCHES = {
    # (scene, pair index, which pixels, which input): depth at the reference pixel, depth at a neighbour tap, normal
    "silhouette taps straddle a hole": ("silhouette", 0, lambda e: e["geo"] & (e["taps_le0"] > 0), "tap"),
    "silhouette reference pixel": ("silhouette", 0, lambda e: e["photo"] & (e["taps_le0"] > 0), "depth"),
    "|n| < eps": ("degenerate", 0, lambda e: e["photo"] & (e["nlen"] < 1e-12), "normal"),
    "|n| < eps depth": ("degenerate", 0, lambda e: e["photo"] & (e["nlen"] < 1e-12), "depth"),
    "|d| small": ("degenerate", 0, lambda e: e["photo"] & (e["d"] < 1e-2) & (e["nlen"] > 0.5), "normal"),
    "|d| small depth": ("degenerate", 0, lambda e: e["photo"] & (e["d"] < 5e-2) & (e["nlen"] > 0.5), "depth"),
    "var a var b below the floor": ("flat", 0, lambda e: e["photo"] & (e["va"] * e["vb"] < 1e-8), "normal"),
    "saturated grey": ("flat", 0, lambda e: e["photo"] & (e["va"] > 0.02), "depth"),
}


@pytest.mark.parametrize("branch", list(BRANCHES))
def test_oracle_matches_finite_differences(branch):
    name, b, select, what = BRANCHES[branch]
    d, n, g, cams, pairs, _ = _maps(name)
    pair = [pairs[b]]
    r, nb = pair[0]
    _, _, (e,) = mo.consistency(d, n, g, cams, pair, TAU, info=True)
    H, W = d.shape[2:]
    gb, pb = mo.borderline_edges(e, TAU, W, H, delta=1e-3)
    pix = _sample(select(e) & ~(gb | pb), 6, seed=len(branch))
    counts = [(int(e["geo"].sum()), int(e["photo"].sum()))]
    weights = [e["w"]]
    cot = torch.tensor([0.8, 1.3], dtype=torch.float64)

    def f(dd, nn):
        geo, photo = mo.consistency(dd, nn, g, cams, pair, TAU, counts=counts, weights=weights)
        return geo[0] * cot[0] + photo[0] * cot[1]

    d0, n0 = d.clone().requires_grad_(), n.clone().requires_grad_()
    gd, gn = torch.autograd.grad(f(d0, n0), [d0, n0])
    checked = 0
    for p in pix:
        if what == "normal":
            elems = [(n, gn, (r, c, p // W, p % W)) for c in range(3)]
        elif what == "depth":
            elems = [(d, gd, (r, 0, p // W, p % W))]
        else:                                        # the neighbour taps of q that carry weight
            qx, qy = e["q"][p].tolist()
            x0, y0 = int(qx // 1), int(qy // 1)
            elems = [(d, gd, (nb, 0, y, x)) for y in (y0, y0 + 1) for x in (x0, x0 + 1)
                     if 0 <= x < W and 0 <= y < H and (1 - abs(qx - x)) * (1 - abs(qy - y)) > 1e-3]
        for base, grad, i in elems:
            # a step relative to the element's own scale: a normal's length, or a depth (at least 1e-2 at a hole)
            size = float(n[i[0], :, i[2], i[3]].norm()) if base is n else max(float(base[i].abs()), 1e-2)
            h = 1e-5 * size
            with torch.no_grad():
                up, dn = base.clone(), base.clone()
                up[i] += h
                dn[i] -= h
                fd = (f(up, n) - f(dn, n)) / (2 * h) if base is d else (f(d, up) - f(d, dn)) / (2 * h)
            an = float(grad[i])
            assert abs(float(fd) - an) <= 1e-5 * abs(an) + 1e-6 * float(grad.abs().max()), (branch, i, float(fd), an)
            checked += 1
    assert checked >= 4, (branch, checked)
