"""render64, the fp64 truth of the rasterizer's mode matrix, on the CPU: on lists built here by a brute-force tile
overlap and depth sort, it equals raster64's and raydepth64's recomposites, its gradients equal central differences,
and its pair-leaf absgrad equals absgrad64's closed form.  And the table of backward-compositor instantiations that
test_mode_matrix_gpu.py holds to it covers every one launch_bwd_ng dispatches."""
import math
import os
import re

import pytest
import torch

import absgrad64
import raster64
import raydepth64
import render64
from relightable3dgaussian_b200 import synth

W, H, S = 40, 36, 3
BG = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64)


def _scene(seed=3, P=90):
    """fp64 leaves (SH degree 3) of a shell scene, none of them near the frustum clamp, and the camera."""
    sc = synth.make_scene(4 * P, "shell-v1", seed, S)
    c = synth.make_camera(1, W, H)
    cam = render64.Camera(c.viewmatrix, c.projmatrix, c.campos, W, H, c.tanfovx, c.tanfovy, c.cx, c.cy)
    t = sc.means3D.double() @ cam.V[:3, :3] + cam.V[3, :3]
    inside = ((t[:, 0] / t[:, 2]).abs() < 1.2 * cam.tanfovx) & ((t[:, 1] / t[:, 2]).abs() < 1.2 * cam.tanfovy) & \
        (t[:, 2] > 0.5)
    idx = torch.nonzero(inside)[:P, 0]
    g = torch.Generator().manual_seed(seed)
    shs = 0.3 * torch.randn(idx.numel(), 16, 3, generator=g, dtype=torch.float64)
    lv = dict(means3D=sc.means3D[idx].double(), opacities=sc.opacities[idx].double(), shs=shs,
              scales=2.0 * sc.scales[idx].double(), rotations=sc.rotations[idx].double(),
              features=sc.features[idx].double())
    return lv, cam


def _const(lv, cam, f3d):
    """The SH clamp flags of the fp64 colours (clamped where 0.5 + sum < 0) and a 3D filter."""
    P = lv["means3D"].shape[0]
    const = {"clamped": torch.zeros(P, 3, dtype=torch.float64)}
    if f3d:
        const["filter_3d"] = 0.004 + 0.004 * torch.arange(P, dtype=torch.float64) % 3
    rec = render64.record(lv, const, cam, 3, f3d=f3d)
    const["clamped"] = (rec[:, 7:10] < 0).double()
    return const


def _state(rec, cam):
    """The kernel's forward state, brute force in fp64: the reference's 3-sigma tile rectangle, the (tile, depth)
    sort, and n_contrib from a front-to-back walk with the forward's skip and stop tests."""
    P = rec.shape[0]
    ndc, tz, conic, op = rec[:, 0:2], rec[:, 2], rec[:, 3:6], rec[:, 6]
    mean2D = ((ndc + 1.0) * torch.tensor([W, H], dtype=torch.float64) - 1.0) * 0.5
    a, b, c = conic.unbind(1)
    det = a * c - b * b
    ca, cb, cc = c / det, -b / det, a / det                          # cov2D from the conic
    mid = 0.5 * (ca + cc)
    lam = mid + torch.sqrt((mid * mid - (ca * cc - cb * cb)).clamp_min(0.1))
    r = torch.ceil(3.0 * torch.sqrt(lam))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    x0 = ((mean2D[:, 0] - r) / 16).floor().clamp(0, gx).long()
    x1 = ((mean2D[:, 0] + r + 15) / 16).floor().clamp(0, gx).long()
    y0 = ((mean2D[:, 1] - r) / 16).floor().clamp(0, gy).long()
    y1 = ((mean2D[:, 1] + r + 15) / 16).floor().clamp(0, gy).long()
    keys = []
    for i in range(P):
        if tz[i] <= 0.2:
            continue
        for ty in range(int(y0[i]), int(y1[i])):
            for tx in range(int(x0[i]), int(x1[i])):
                keys.append((ty * gx + tx, float(tz[i]), i))
    keys.sort()
    point_list = torch.tensor([k[2] for k in keys], dtype=torch.long)
    tile = torch.tensor([k[0] for k in keys], dtype=torch.long)
    ranges = torch.zeros(gx * gy, 2, dtype=torch.long)
    for t in range(gx * gy):
        hit = torch.nonzero(tile == t)[:, 0]
        if hit.numel():
            ranges[t] = torch.tensor([int(hit[0]), int(hit[-1]) + 1])
    st = dict(point_list=point_list, ranges=ranges, means2D=mean2D, conic_opacity=torch.cat([conic, op[:, None]], 1),
              rgb=rec[:, 7:10], depths=tz)
    # n_contrib: a walk over the whole tile list (n_contrib = the list length for the moment)
    full = torch.zeros(H, W, dtype=torch.long)
    for y in range(H):
        for x in range(W):
            t = (y // 16) * gx + x // 16
            full[y, x] = ranges[t, 1] - ranges[t, 0]
    wk = raster64.Walk(dict(st, n_contrib=full), list(range(gx * gy)), W, H)
    one = 1.0 - wk.alpha
    stop = wk.valid & (wk.T * one < raster64.T_CUT)
    before = torch.cumsum(stop.long(), 1) - stop.long() == 0
    comp = wk.valid & before & ~stop
    j = torch.arange(1, comp.shape[1] + 1)
    nc = torch.zeros(H * W, dtype=torch.long)
    nc[wk.pix] = torch.where(comp, j[None, :], torch.zeros_like(j)[None, :]).amax(1)
    st["n_contrib"] = nc.view(H, W)
    return st


def _setup(aa=False, f3d=False, seed=3):
    lv, cam = _scene(seed)
    const = _const(lv, cam, f3d)
    rec = render64.record(lv, const, cam, 3, aa=aa, f3d=f3d)
    st = _state(rec, cam)
    st["features"] = lv["features"]
    return lv, const, cam, rec, st


def test_brute_force_lists_are_long_enough():
    _, _, _, _, st = _setup()
    nc = st["n_contrib"]
    assert int(nc.max()) >= 10 and float((nc > 0).double().mean()) > 0.3


@pytest.mark.parametrize("aa,f3d", [(False, False), (True, True)])
def test_modes_off_equal_the_raster64_recomposite(aa, f3d):
    lv, const, cam, rec, st = _setup(aa, f3d)
    out = render64.render(lv, const, cam, st, BG, D=3, aa=aa, f3d=f3d)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    wk = raster64.Walk(st, list(range(gx * gy)), W, H)
    want = wk.composite(st, BG, S, wk.alpha)                          # [n, 3 + 1 + 1 + S]
    got = torch.cat([out.images[k].reshape(-1 if k in ("opacity", "depth") else out.images[k].shape[0], H * W).T
                     .reshape(H * W, -1) for k in ("color", "opacity", "depth", "feature")], 1)[wk.pix]
    err = (got - want).abs().max() / want.abs().max()
    assert float(err) <= 1e-12, float(err)


def test_ray_depth_equals_the_raydepth64_composite():
    lv, const, cam, rec, st = _setup()
    out = render64.render(lv, const, cam, st, BG, D=3, ray_depth=True)
    gx = (W + 15) // 16
    nc = st["n_contrib"].reshape(-1)
    order = []
    for pix in range(H * W):
        t = (pix // W // 16) * gx + (pix % W) // 16
        order.append(st["point_list"][st["ranges"][t, 0]:st["ranges"][t, 1]])
    want = raydepth64.composite_depth(st["means2D"], rec[:, 3:6], rec[:, 6], rec[:, 2], rec[:, 10:12], order, nc, W, H)
    err = (out.images["depth"][0] - want).abs().max() / want.abs().max()
    assert float(err) <= 1e-12, float(err)


def _cots(out, seed=1):
    g = torch.Generator().manual_seed(seed)
    live = (~out.ambiguous_pixels()).double()
    return {k: torch.randn(v.shape, generator=g, dtype=torch.float64) * live for k, v in out.images.items()}


def test_gradients_against_central_differences():
    """Every mode on (AA, 3D filter, ray depth, depth statistics, surface outputs): autograd of a few leaf entries, camera
    entries and pair leaves against central differences of the same fp64 map."""
    aa = f3d = rd = ds = surf = True
    lv, const, cam0, rec, st = _setup(aa, f3d)
    cam_leaves = {k: getattr(cam0, a).clone() for k, a in (("viewmatrix", "V"), ("projmatrix", "P"),
                                                            ("campos", "campos"))}
    kw = dict(D=3, aa=aa, f3d=f3d, ray_depth=rd, depth_stats=ds, surface=surf)

    def loss_of(lv_, cl, cots=None, shift=None):
        cam = render64.Camera(cl["viewmatrix"], cl["projmatrix"], cl["campos"], W, H, cam0.tanfovx, cam0.tanfovy,
                              cam0.cx, cam0.cy)
        out = render64.render(lv_, const, cam, st, BG, shift=shift, **kw)
        cots = _cots(out) if cots is None else cots
        return sum((out.images[k] * c).sum() for k, c in cots.items()), out, cots

    P = lv["means3D"].shape[0]
    lv = dict(lv, off=torch.zeros(P, 3, dtype=torch.float64))
    leaves = {k: v.clone().requires_grad_(True) for k, v in lv.items()}
    cl = {k: v.clone().requires_grad_(True) for k, v in cam_leaves.items()}
    loss, out, cots = loss_of(leaves, cl)
    assert float(out.ambiguous_pixels().double().mean()) < 0.05
    names = list(leaves) + list(cl)
    grads = torch.autograd.grad(loss, [leaves[k] for k in leaves] + [cl[k] for k in cl] + out.pair_leaves(),
                                allow_unused=True)
    gd = dict(zip(names, grads[:len(names)]))
    pg = grads[len(names):]
    # the rows most composited, and one entry of each leaf
    _, ids, keep = out.pairs[0]
    busy = torch.bincount(ids[keep], minlength=P).argsort(descending=True)[:2].tolist()
    probes = [(k, (i,) + (0,) * (lv[k].dim() - 1)) for i in busy for k in lv]
    probes += [(k, (i, 1)) for i in busy for k in ("means3D", "scales", "rotations", "off")]
    probes += [("viewmatrix", (0, 0)), ("viewmatrix", (2, 1)), ("viewmatrix", (3, 2)), ("projmatrix", (1, 1)),
               ("projmatrix", (3, 0)), ("campos", (1,))]
    h = 1e-6
    fails = []
    for k, at in probes:
        def f(sgn):
            lv2 = {n: v.clone() for n, v in lv.items()}
            cl2 = {n: v.clone() for n, v in cam_leaves.items()}
            (lv2 if k in lv2 else cl2)[k][at] += sgn * h
            return float(loss_of(lv2, cl2, cots)[0])
        fd = (f(1) - f(-1)) / (2 * h)
        ad = float(gd[k][at]) if gd[k] is not None else 0.0
        if abs(fd - ad) > 1e-5 * max(abs(ad), 1e-3 * float(gd[k].abs().max())):
            fails.append((k, at, ad, fd))
    # pair leaves: the two largest pairs
    g0 = pg[0][..., :2].reshape(-1, 2)
    for flat in g0.abs().amax(1).argsort(descending=True)[:2].tolist():
        i, j = divmod(flat, pg[0].shape[1])
        for c in range(2):
            v = torch.zeros(2, dtype=torch.float64)
            v[c] = h
            fd = (float(loss_of(lv, cam_leaves, cots, {(0, i, j): v})[0]) -
                  float(loss_of(lv, cam_leaves, cots, {(0, i, j): -v})[0])) / (2 * h)
            ad = float(pg[0][i, j, c])
            if abs(fd - ad) > 1e-5 * abs(ad):
                fails.append(("pair", (i, j, c), ad, fd))
    assert not fails, fails
    # the pairs' gradients sum to the mean's
    sums = torch.zeros(P, 2, dtype=torch.float64)
    for (_, ids_, keep_), g in zip(out.pairs, pg):
        sums.index_add_(0, ids_[keep_], g[keep_][:, :2])
    assert float((sums - gd["off"][:, :2]).abs().max()) <= 1e-12 * float(sums.abs().max())
    # and their opacity terms, with the leaf's factor, to the opacity's gradient, whose magnitude they bound
    op = torch.zeros(P, dtype=torch.float64)
    for (_, ids_, keep_), g in zip(out.pairs, pg):
        op.index_add_(0, ids_[keep_], g[keep_][:, 2])
    want = gd["opacities"].reshape(-1)
    assert float((op * out.op_factor - want).abs().max()) <= 1e-12 * float(want.abs().max())
    assert bool((out.opacity_magnitude(pg) >= want.abs() * (1 - 1e-12)).all())


@pytest.mark.parametrize("aa", [False, True])
def test_absgrad_equals_the_closed_form(aa):
    lv, const, cam, rec, st = _setup(aa)
    out = render64.render(lv, const, cam, st, BG, D=3, aa=aa)
    cots = _cots(out, seed=2)
    loss = sum((out.images[k] * c).sum() for k, c in cots.items())
    pg = torch.autograd.grad(loss, out.pair_leaves())
    got = out.absgrad(pg)
    st64 = dict(st, conic_opacity=torch.cat([rec[:, 3:6], rec[:, 6:7]], 1))
    want, _ = absgrad64.row_truth(st64, absgrad64.walks_of(st64, W, H), [cots[k] for k in ("color", "opacity", "depth",
                                                                                          "feature")], BG, W, H, S)
    assert float(want.abs().max()) > 0
    err = (got - want).abs().max() / want.abs().max()
    assert float(err) <= 1e-12, float(err)


# ---- the dispatch table ---------------------------------------------------------------------------------------------
def _dispatched():
    """The (DET, GEOM, ABS, RD, DS) tuples launch_bwd_ng in composite_bwd.cu instantiates, template defaults filled."""
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "relightable3dgaussian_b200",
                        "csrc", "composite_bwd.cu")
    src = open(path).read()
    head = re.search(r"template\s*<int NG, bool DET, bool GEOM((?:, bool \w+ = (?:true|false))*)>\s*"
                     r"static void launch_bwd_kernel", src)
    assert head, "launch_bwd_kernel's template head not found"
    defaults = [d == "true" for d in re.findall(r"= (true|false)", head.group(1))]
    body = re.search(r"static void launch_bwd_ng\([^)]*\)\s*\{(.*?)\n\}", src, re.S)
    assert body, "launch_bwd_ng not found"
    found = set()
    for args in re.findall(r"launch_bwd_kernel<NG,\s*([^>]*)>", body.group(1)):
        vals = [a.strip() == "true" for a in args.split(",")]
        found.add(tuple(vals + defaults[len(vals) - 2:]))
    return found


def test_every_dispatched_backward_kernel_has_a_truth_case():
    import test_mode_matrix_gpu as mm
    found = _dispatched()
    assert len(found) >= 18, found
    table = set(mm.KERNELS)
    assert found <= table, sorted(found - table)
    assert table <= found, sorted(table - found)


def test_mode_matrix_channel_counts_cover_every_group():
    import test_mode_matrix_gpu as mm
    groups = sorted({math.ceil((3 + s) / 4) for s in mm.CHANNELS})
    assert groups == list(range(1, 8)), groups
    assert {17, 18} <= set(mm.CHANNELS)             # both sides of the E = 16 / E = 8 switch (NG 5 and 6)
