"""The bilateral-grid slice on the GPU (bilagrid.slice, csrc/bilagrid.cu) against the fp64 truth of
tests/bilagrid_oracle.py: outputs and both gradients, batches with repeated ids, bitwise reproducibility, gradient
routing, the chain from rasterize_views, and a short fit of known per-image colour transforms."""
import numpy as np
import pytest
import torch

import bilagrid_oracle as bo
from relightable3dgaussian_b200 import bilagrid, synth
from relightable3dgaussian_b200.rasterizer import GaussianRasterizationSettings, rasterize_views

pytestmark = pytest.mark.gpu


def run(grids, rgb, ids, dout, need_grids=True, need_rgb=True):
    g = grids.cuda().requires_grad_(need_grids)
    x = rgb.cuda().requires_grad_(need_rgb)
    out = bilagrid.slice(g, x, ids)
    out.backward(dout.cuda())
    return out.detach(), (x.grad if need_rgb else None), (g.grad if need_grids else None)


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def test_identity_grid_returns_rgb_bitwise():
    m = bilagrid.BilateralGrid(3).cuda()
    rgb = (torch.rand(2, 3, 160, 212, device="cuda") * 1.6 - 0.3)      # luma below 0 and above 1 included
    out = m(rgb, [2, 0])
    assert bits_equal(out, rgb)
    one = rgb[1]
    assert bits_equal(m(one, 1), one)


@pytest.mark.parametrize("H,W", [(800, 800), (1200, 1600)])
def test_matches_fp64_truth(H, W):
    grids, rgb = bo.random_case(2, 1, H, W, seed=H, luma_lo=-0.1, luma_hi=1.1, noise=0.2)
    dout = np.random.default_rng(1).standard_normal(rgb.shape).astype(np.float32)
    out, drgb, dgrids = run(torch.from_numpy(grids), torch.from_numpy(rgb), [1], torch.from_numpy(dout))
    out64 = bo.slice64(grids, rgb, [1])
    drgb64, dgrids64, iz = bo.grads64(grids, rgb, [1], dout)
    err = np.abs(out.cpu().numpy() - out64)
    assert err.max() <= 4e-6 * max(np.abs(out64).max(), 1.0), err.max()
    keep = ~bo.near_node_mask(iz, 8)[:, None]
    err = np.abs(np.where(keep, drgb.cpu().numpy() - drgb64, 0))
    assert err.max() <= 1e-5 * np.abs(drgb64).max(), err.max()
    err = np.abs(dgrids.cpu().numpy() - dgrids64)
    assert err.max() <= 1e-5 * np.abs(dgrids64).max(), err.max()
    assert np.all(dgrids.cpu().numpy()[0] == 0)                 # grid 0 is not used


def test_luma_clamp_rule():
    """Luma well below 0 or above 1 in whole image rows: the luma term is exactly absent, dL/drgb = A^T dL/dout; rows in
    between keep it.  No pixel lies near a node, so the comparison needs no mask."""
    H, W, L = 96, 128, 8
    grids, _ = bo.random_case(1, 1, H, W, L, seed=5, noise=0.3)
    rs = np.random.default_rng(2)
    rgb = np.empty((1, 3, H, W), np.float32)
    rgb[:, :, :32] = rs.uniform(-0.8, -0.2, (1, 3, 32, W))
    rgb[:, :, 32:64] = rs.uniform(1.2, 1.8, (1, 3, 32, W))
    rgb[:, :, 64:] = rs.uniform(0.2, 0.8, (1, 3, 32, W))
    dout = rs.standard_normal(rgb.shape).astype(np.float32)
    _, drgb, _ = run(torch.from_numpy(grids), torch.from_numpy(rgb), [0], torch.from_numpy(dout), need_grids=False)
    drgb64, _, iz = bo.grads64(grids, rgb, [0], dout)
    A = bo.affine(grids[0].astype(np.float64), rgb[0].astype(np.float64)).reshape(3, 4, H, W)
    affine_only = np.einsum("cjhw,chw->jhw", A[:, :3], dout[0].astype(np.float64))
    d = drgb.cpu().numpy()[0]
    scale = np.abs(drgb64).max()
    assert np.abs(d[:, :64] - affine_only[:, :64]).max() <= 1e-5 * scale
    mid = bo.near_node_mask(iz, L)[0, 64:]
    assert not mid.any()
    assert np.abs(d[:, 64:] - drgb64[0, :, 64:]).max() <= 1e-5 * scale
    assert np.abs(drgb64[0, :, 64:] - affine_only[:, 64:]).max() > 10 * 1e-5 * scale     # the luma term is there


def test_batch_with_repeated_ids_equals_one_view_calls():
    ids = [2, 0, 2, 1, 2]
    grids, rgb = bo.random_case(4, len(ids), 200, 240, seed=9, noise=0.2)
    dout = np.random.default_rng(3).standard_normal(rgb.shape).astype(np.float32)
    g, x, d = map(torch.from_numpy, (grids, rgb, dout))
    out, drgb, dgrids = run(g, x, ids, d)
    parts = []
    for n, i in enumerate(ids):
        o1, dr1, dg1 = run(g, x[n:n + 1], [i], d[n:n + 1])
        assert bits_equal(out[n:n + 1], o1), n
        assert bits_equal(drgb[n:n + 1], dr1), n
        parts.append(dg1)
    want = sum(parts)
    assert torch.all(dgrids[3] == 0)
    assert (dgrids - want).abs().max() <= 1e-6 * want.abs().max()


def test_reproducible_and_unchanged_under_deterministic_algorithms():
    grids, rgb = bo.random_case(2, 3, 300, 420, seed=4, noise=0.2)
    dout = np.random.default_rng(4).standard_normal(rgb.shape).astype(np.float32)
    args = (torch.from_numpy(grids), torch.from_numpy(rgb), [1, 0, 1], torch.from_numpy(dout))
    a, b = run(*args), run(*args)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        c = run(*args)
    finally:
        torch.use_deterministic_algorithms(prev)
    for x, y, z in zip(a, b, c):
        assert bits_equal(x, y) and bits_equal(x, z)


def test_gradient_routing_and_non_contiguous_input():
    grids, rgb = bo.random_case(2, 2, 130, 170, seed=6, noise=0.2)
    dout = np.random.default_rng(6).standard_normal(rgb.shape).astype(np.float32)
    g, x, d = map(torch.from_numpy, (grids, rgb, dout))
    out, drgb, dgrids = run(g, x, [1, 0], d)
    _, drgb_only, none = run(g, x, [1, 0], d, need_grids=False)
    assert none is None and bits_equal(drgb_only, drgb)
    _, none, dgrids_only = run(g, x, [1, 0], d, need_rgb=False)
    assert none is None and bits_equal(dgrids_only, dgrids)
    # a channels-last view: the same pixels through a non-contiguous tensor
    xs = x.cuda().permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2).requires_grad_(True)
    assert not xs.is_contiguous()
    gg = g.cuda().requires_grad_(True)
    o2 = bilagrid.slice(gg, xs, [1, 0])
    o2.backward(d.cuda())
    assert bits_equal(o2, out) and bits_equal(xs.grad.contiguous(), drgb) and bits_equal(gg.grad, dgrids)


def test_refusals_on_the_gpu():
    g = bilagrid.BilateralGrid(2, 4, 4, 2).cuda().grids
    x = torch.rand(3, 64, 64, device="cuda", requires_grad=True)
    with pytest.raises(ValueError, match="CUDA"):
        bilagrid.slice(g, x.detach().cpu(), 0)
    with pytest.raises(ValueError, match="CPU"):
        bilagrid.slice(g, x, torch.tensor([0], device="cuda"))
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="devices"):
            bilagrid.slice(g, x.detach().to("cuda:1"), 0)
    out = bilagrid.slice(g, x, 1)
    (dx,) = torch.autograd.grad(out.sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        dx.sum().backward()


def _scene(V, W=160, H=120, P=3000):
    sc = synth.make_scene(P, seed=0, S=0)
    settings = []
    for k in range(V):
        cam = synth.make_camera(k, W, H)
        settings.append(GaussianRasterizationSettings(H, W, cam.tanfovx, cam.tanfovy, cam.cx, cam.cy,
                                                      torch.tensor([0.2, 0.3, 0.4]).cuda(), 1.0, cam.viewmatrix.cuda(),
                                                      cam.projmatrix.cuda(), 3, cam.campos.cuda(), False, True, True,
                                                      False))
    leaves = {k: getattr(sc, k).cuda().contiguous().requires_grad_(True)
              for k in ("means3D", "opacities", "shs", "scales", "rotations")}
    return settings, leaves


def test_rasterize_views_then_slice_then_l1_matches_the_torch_chain():
    V, ids = 2, [1, 0]
    settings, leaves = _scene(V)
    grids, _ = bo.random_case(2, 1, 8, 8, seed=8, noise=0.1)
    grids = torch.from_numpy(grids).cuda()
    target = torch.rand(V, 3, 120, 160, device="cuda")
    grads = []
    for fn in (lambda gr, img: bilagrid.slice(gr, img, ids), lambda gr, img: bo.torch_slice(gr, img, ids)):
        for t in leaves.values():
            t.grad = None
        gr = grids.clone().requires_grad_(True)
        m2d = torch.zeros(V, leaves["means3D"].shape[0], 3, device="cuda", requires_grad=True)
        out = rasterize_views(leaves["means3D"], m2d, leaves["opacities"], settings=settings, shs=leaves["shs"],
                              scales=leaves["scales"], rotations=leaves["rotations"])
        color = out[2]
        loss = (fn(gr, color) - target).abs().mean()
        loss.backward()
        grads.append({k: t.grad.clone() for k, t in leaves.items()} | {"grids": gr.grad.clone()})
    for k in grads[0]:
        a, b = grads[0][k], grads[1][k]
        assert a.abs().max() > 0, k
        rel = ((a - b).norm() / b.norm()).item()
        assert rel < 2e-3, (k, rel)


def test_adam_fits_known_per_image_affine_changes():
    torch.manual_seed(0)
    H, W = 96, 128
    rgb = torch.rand(2, 3, H, W, device="cuda")
    M = torch.tensor([[[1.2, 0.1, 0.0], [0.0, 0.9, 0.05], [0.05, 0.0, 0.8]],
                      [[0.8, 0.0, 0.1], [0.1, 1.1, 0.0], [0.0, 0.1, 1.15]]], device="cuda")
    b = torch.tensor([[0.05, -0.02, 0.1], [-0.05, 0.03, 0.0]], device="cuda")
    target = torch.einsum("ncj,njhw->nchw", M, rgb) + b[:, :, None, None]
    m = bilagrid.BilateralGrid(2, 8, 8, 4).cuda()
    opt = torch.optim.Adam(m.parameters(), lr=2e-2)
    losses = []
    for _ in range(60):
        opt.zero_grad()
        loss = (m(rgb, [0, 1]) - target).abs().mean()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.2 * losses[0], losses[::10]
