"""Multi-view consistency losses on the GPU against the fp64 oracle on adversarial maps (tests/multiview_edges.py), in
the default and the deterministic gradient mode: branch coverage per scene, losses and counts, every gradient element
off the borderline pixels, exact zeros where the definition has no term, the forward's and the backward's pixel sets,
bitwise reproducibility under repetition and pair permutation, extreme cotangents and thresholds, and scale."""
import pytest
import torch

import multiview_edges as me
import multiview_oracle as mo
from multiview_check import DEV, TAU, Truth, _kernel, _rel, _settings, check_losses, check_pixels, det_resolution

pytestmark = pytest.mark.gpu
MODES = (False, True)
_SCENES = {}


def _scene(name):
    """(depth, normal, gray) float32 on the device, cams, settings, pairs and coverage of a scene (built once)."""
    if name not in _SCENES:
        build, pairs, cov = me.SCENES[name]
        depth, normal, gray, cams = build()
        d, n, g = (t.float().to(DEV).contiguous() for t in (depth, normal, gray))
        _SCENES[name] = (d, n, g, cams, _settings(cams, d.shape[3], d.shape[2]), pairs, cov)
    return _SCENES[name]


def _cot(B, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return tuple(scale * (torch.rand(B, device=DEV, generator=g) + 0.5) for _ in range(2))


def _run(d, n, g, settings, pairs, cot, det, tau=TAU):
    torch.use_deterministic_algorithms(det)
    try:
        return _kernel(d, n, g, settings, pairs, cot, tau)
    finally:
        torch.use_deterministic_algorithms(False)


def _check_modes(name, d, n, g, cams, settings, pairs, cot, tau=TAU):
    """Both modes against one fp64 truth; returns (truth, {mode: kernel outputs}, {mode: worst elements})."""
    k0 = _run(d, n, g, settings, pairs, cot, False, tau)
    t = Truth(d, n, g, cams, pairs, cot, k0[2], tau)
    out, worst = {}, {}
    for det in MODES:
        k = k0 if not det else _run(d, n, g, settings, pairs, cot, True, tau)
        assert torch.equal(k[2], k0[2]) and torch.equal(k[0], k0[0]) and torch.equal(k[1], k0[1])
        label = (name, "deterministic" if det else "default")
        check_losses(k[:3], t, label)
        worst[det] = check_pixels(k[3], k[4], t, label, det_resolution(cot, k0[2]) if det else 0.0)
        out[det] = k
    return t, out, worst


@pytest.mark.parametrize("name", list(me.SCENES))
def test_scene_against_fp64(name):
    d, n, g, cams, settings, pairs, cov = _scene(name)
    cot = _cot(len(pairs), 11)
    t, out, worst = _check_modes(name, d, n, g, cams, settings, pairs, cot)
    coverage = cov(t.info, (d.double(), n.double(), g.double(), cams))
    for branch, (count, least) in coverage.items():
        assert count >= least, (name, branch, count, least)
    print(f"\nREPORT {name} coverage={ {k: v[0] for k, v in coverage.items()} } border={t.border} kinks={t.kinks} "
          f"worst_default={worst[False]} worst_det={worst[True]}")
    # deterministic mode: bitwise under repetition and under a permutation of the pairs (gradients are per-view sums)
    kd = out[True]
    again = _run(d, n, g, settings, pairs, cot, True)
    perm = torch.randperm(len(pairs), generator=torch.Generator().manual_seed(3)).tolist()
    permuted = _run(d, n, g, settings, [pairs[i] for i in perm], tuple(c[perm] for c in cot), True)
    for x, y, z in zip(kd[3:], again[3:], permuted[3:]):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
        assert torch.equal(x.view(torch.int32), z.view(torch.int32))
    assert torch.equal(permuted[0], kd[0][perm]) and torch.equal(permuted[2], kd[2][perm])


@pytest.mark.parametrize("name", [k for k in me.SCENES if not k.startswith(("tiny", "scale"))] + ["tiny15x16"])
@pytest.mark.parametrize("det", MODES, ids=["default", "deterministic"])
def test_forward_and_backward_agree_on_the_pixel_set(name, det):
    """For each pair alone (r != n): the reference pixels with a nonzero dL/ddepth under a geo-only cotangent are
    the forward's geo-valid pixels, and those with a nonzero dL/dnormal under a photo-only cotangent the photo-valid
    ones (the forward and the backward are separate instantiations of the pixel code)."""
    d, n, g, cams, settings, pairs, _ = _scene(name)
    one = torch.ones(1, device=DEV)
    for r, nb in sorted({p for p in pairs if p[0] != p[1]})[:4]:
        with torch.no_grad():
            _, _, (e,) = mo.consistency(d.double(), n.double(), g.double(), cams, [(r, nb)], TAU, info=True)
        kg = _run(d, n, g, settings, [(r, nb)], (one, None), det)
        n_geo = int(kg[2][0, 0])
        nz = int((kg[3][r, 0] != 0).sum())
        phi0 = int((e["geo"] & (e["phi"] == 0)).sum())
        assert n_geo - phi0 <= nz <= n_geo, (name, (r, nb), nz, n_geo, phi0)
        kp = _run(d, n, g, settings, [(r, nb)], (None, one), det)
        n_photo = int(kp[2][0, 1])
        nz = int((kp[4][r] != 0).any(0).sum())
        flat = int((e["photo"] & (1 - e["ncc"] < 0)).sum())
        assert n_photo - flat <= nz <= n_photo, (name, (r, nb), nz, n_photo, flat)


CASES = {
    "geo None": lambda c: (None, c[1]), "photo None": lambda c: (c[0], None),
    "geo zero": lambda c: (torch.zeros_like(c[0]), c[1]), "photo zero": lambda c: (c[0], torch.zeros_like(c[1])),
    "pair 0 zero": lambda c: (torch.cat([c[0][:1] * 0, c[0][1:]]), torch.cat([c[1][:1] * 0, c[1][1:]])),
    "1e-8": lambda c: (c[0] * 1e-8, c[1] * 1e-8), "1e4": lambda c: (c[0] * 1e4, c[1] * 1e4),
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("name", ["silhouette", "degenerate"])
def test_cotangent_extremes(name, case):
    d, n, g, cams, settings, pairs, _ = _scene(name)
    _check_modes((name, case), d, n, g, cams, settings, pairs, CASES[case](_cot(len(pairs), 5)))


def test_threshold_zero_and_huge():
    d, n, g, cams, settings, pairs, _ = _scene("silhouette")
    cot = _cot(len(pairs), 6)
    for det in MODES:
        kg, kp, counts, gd, gn = _run(d, n, g, settings, pairs, cot, det, tau=0.0)
        assert bool((kg == 0).all()) and bool((kp == 0).all()) and bool((counts == 0).all())
        assert bool((gd == 0).all()) and bool((gn == 0).all())
    t, out, _ = _check_modes("tau 1e30", d, n, g, cams, settings, pairs, cot, tau=1e30)
    assert int(out[False][2][:, 0].min()) > int(t.info[0]["geo"].numel() * 0.5)


def test_scale_equivariance():
    """geo, photo and the counts of the 1e-3 and 1e3 scenes agree with the unit scene's within the fp64 oracle's own
    differences, and dL/ddepth scales as 1 / s (each scale is held to the fp64 truth in test_scene_against_fp64)."""
    res = {}
    for x in me.SCALES:
        d, n, g, cams, settings, pairs, _ = _scene(f"scale{x:g}")
        res[x] = _check_modes(("scale", x), d, n, g, cams, settings, pairs, _cot(len(pairs), 12))[:2]
    t1, out1 = res[1.0]
    V = t1.V
    for s in (x for x in me.SCALES if x != 1.0):
        t, out = res[s]
        for det in MODES:
            k, k1 = out[det], out1[det]
            for i, key in enumerate(("geo", "photo")):
                tv, tv1, fv, fv1 = (t.tg, t1.tg, t.fg, t1.fg) if i == 0 else (t.tp, t1.tp, t.fp, t1.fp)
                for b in range(len(t.info)):
                    nb = t.border[b][i] + t1.border[b][i]
                    slack = abs(float(tv[b]) - float(tv1[b])) + 4 * (abs(float(fv[b] - tv[b])) + abs(float(fv1[b] - tv1[b])))
                    assert abs(float(k[i][b]) - float(k1[i][b])) <= slack + nb / max(int(k[2][b, i]), 1) + 1e-6, \
                        (s, det, key, b, float(k[i][b]), float(k1[i][b]), slack)
                    want = abs(int(t.info[b][key].sum()) - int(t1.info[b][key].sum()))
                    assert abs(int(k[2][b, i]) - int(k1[2][b, i])) <= want + nb, (s, det, key, b)
            keep = ~(t.skip | t1.skip)
            rk = _rel(k[3].reshape(V, -1) * s, k1[3].reshape(V, -1), keep)
            rt = _rel(t.gd.reshape(V, -1) * s, t1.gd.reshape(V, -1), keep)
            rf = _rel(t.fgd.reshape(V, -1), t.gd.reshape(V, -1), keep) + _rel(t1.fgd.reshape(V, -1), t1.gd.reshape(V, -1),
                                                                                keep)
            assert rk <= rt + 4 * rf + 1e-6, (s, det, rk, rt, rf)


def test_closed_image_bound():
    """q exactly on the last column and row is inside the image ([0, W-1] x [0, H-1] is closed): an axis-aligned
    camera with fx = fy = 1 and a principal point at 0 reprojects every pixel of (v, v) exactly onto itself."""
    W, H = 20, 12
    cam = mo.Cam(torch.eye(4), W / 2, H / 2, 0.0, 0.0)
    d = torch.full((1, 1, H, W), 2.0, device=DEV)
    n = torch.zeros(1, 3, H, W, device=DEV)
    n[:, 2] = 1.0
    g = torch.rand(1, 1, H, W, generator=torch.Generator().manual_seed(0)).to(DEV)
    for det in MODES:
        kg, kp, counts, gd, gn = _run(d, n, g, _settings([cam], W, H), [(0, 0)], _cot(1, 1), det)
        assert counts[0].tolist()[0] == W * H and float(kg[0]) == 0.0
