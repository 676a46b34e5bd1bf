"""GPU parity of the fused SSIM loss (relightable3dgaussian_b200.losses.ssim) against the reference
formula in fp64.  e_kernel is the fused result's error against that truth, e_ref the error of the
IEEE fp32 reference formula (the fixture's fp32 record, or tests/ssim_oracle.py in fp32 on the
GPU).  Values pass at e_kernel <= max(2e-7, 4 e_ref) (absolute), gradients by relative L2 at
<= max(2e-6, 4 e_ref)."""
import os

import numpy as np
import pytest
import torch

import ssim_oracle as oss
from helpers import GOLDEN, npy, rel_l2

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(GOLDEN, "ssim.npz"))


def fused(a, b, size_average):
    from relightable3dgaussian_b200.losses import ssim
    return ssim(a, b, size_average=size_average)


def ours(a, b, cot, size_average):
    v, g1, g2 = oss.value_and_grads(fused, a.cuda(), b.cuda(), cot.cuda(), size_average, torch.float32)
    return npy(v), npy(g1), npy(g2)


def check(tag, mine, truth, ref32, identical=False):
    """mine / truth / ref32: (value, dL/dimg1, dL/dimg2).  Returns the ratios e_kernel / e_ref."""
    ek = np.abs(np.float64(mine[0]) - truth[0]).max()
    er = np.abs(np.float64(ref32[0]) - truth[0]).max()
    assert ek <= max(2e-7, 4 * er), (tag, "value", ek, er)
    ratios = [ek / max(er, 1e-30)]
    for i in (1, 2):
        if identical:      # the true gradient is 0: compare absolute L2 norms of the rounding noise
            ek, er = (np.linalg.norm(np.float64(x[i]) - truth[i]) for x in (mine, ref32))
            floor = 1e-7
        else:
            ek, er, floor = rel_l2(mine[i], truth[i]), rel_l2(ref32[i], truth[i]), 2e-6
        assert ek <= max(floor, 4 * er), (tag, f"grad{i}", ek, er)
        ratios.append(ek / max(er, 1e-30))
    print(f"[ssim] {tag:34s} e_kernel/e_ref value {ratios[0]:.2f} grad1 {ratios[1]:.2f} grad2 {ratios[2]:.2f}")
    return ratios


@pytest.mark.parametrize("case", oss.GOLDEN_CASES, ids=[c[0] for c in oss.GOLDEN_CASES])
def test_matches_reference_function_golden(case):
    name, kind, shape, size_average, seed = case
    a, b, cot = oss.ssim_case(kind, shape, seed)
    mine = ours(a, b, cot, size_average)
    truth = tuple(G[f"{name}/{k}64"] for k in ("value", "grad1_", "grad2_"))
    ref32 = tuple(G[f"{name}/{k}32"] for k in ("value", "grad1_", "grad2_"))
    assert mine[0].shape == truth[0].shape
    check(name, mine, truth, ref32, identical=kind == "identical")


SIZES = [(3, 800, 800), (3, 1200, 1600), (3, 1080, 1920), (4, 3, 256, 256)]


@pytest.mark.parametrize("kind", ["uniform", "smooth", "nearconst", "rendered"])
@pytest.mark.parametrize("shape", SIZES, ids=["x".join(map(str, s)) for s in SIZES])
def test_matches_ieee_oracle_at_training_sizes(shape, kind):
    a, b, cot = oss.ssim_case(kind, shape, seed=21)
    a, b, cot = a.cuda(), b.cuda(), cot.cuda()
    size_average = len(shape) == 3
    fn = lambda x, y, sa: oss.ssim(x, y, size_average=sa)
    truth = [npy(t) for t in oss.value_and_grads(fn, a, b, cot, size_average, torch.float64)]
    ref32 = [npy(t) for t in oss.value_and_grads(fn, a, b, cot, size_average, torch.float32)]
    check(f"{kind} {shape}", ours(a, b, cot, size_average), truth, ref32)


def test_identical_images_give_exactly_one():
    a, _, _ = oss.ssim_case("rendered", (3, 1080, 1920), seed=3)
    a = a.cuda()
    assert fused(a, a.clone(), True).item() == 1.0
    b = torch.rand(4, 3, 100, 130, device="cuda")
    assert fused(b, b, True).item() == 1.0
    assert torch.equal(fused(b, b, False), torch.ones(4, device="cuda"))


def test_per_image_values_and_shape():
    a, b, _ = oss.ssim_case("rendered", (5, 3, 70, 90), seed=4)
    a, b = a.cuda(), b.cuda()
    per = fused(a, b, False)
    assert per.shape == (5,) and per.dtype == torch.float32
    ref = oss.ssim(a, b, size_average=False, dtype=torch.float64)
    assert np.abs(npy(per) - npy(ref)).max() < 1e-6
    for n in range(5):
        assert abs(fused(a[n], b[n], True).item() - per[n].item()) < 1e-7
    assert fused(a, b, True).shape == () and fused(a[0], b[0], True).shape == ()


def test_deterministic():
    a, b, cot = oss.ssim_case("uniform", (2, 3, 400, 600), seed=5)
    r1, r2 = ours(a, b, cot, False), ours(a, b, cot, False)
    for x, y in zip(r1, r2):
        assert np.array_equal(x, y)


def test_training_loss_gradient_matches_oracle():
    """(1 - lambda) L1 + lambda (1 - ssim), lambda_dssim = 0.2, as gaussian_renderer/neilf.py:231 builds it."""
    a, b, _ = oss.ssim_case("rendered", (3, 600, 800), seed=6)
    a, b = a.cuda(), b.cuda()
    grads = []
    for fn in (fused, lambda x, y, sa: oss.ssim(x, y, size_average=sa)):
        img = a.clone().requires_grad_(True)
        with oss.ieee_convolutions():
            loss = 0.8 * (img - b).abs().mean() + 0.2 * (1.0 - fn(img, b, True))
            loss.backward()
        grads.append(npy(img.grad))
    assert rel_l2(grads[0], grads[1]) < 1e-5


def test_non_contiguous_views_and_gradient_routing():
    """The eval scripts pass `split` slices; only the requested gradients are computed."""
    from relightable3dgaussian_b200 import _lib
    big = torch.rand(3, 64, 2 * 96, device="cuda", requires_grad=True)
    a, b = big.split(96, dim=-1)
    assert not a.is_contiguous()
    v = fused(a, b, True)
    ac, bc = a.detach().contiguous().requires_grad_(True), b.detach().contiguous().requires_grad_(True)
    vc = fused(ac, bc, True)
    assert torch.equal(v, vc)
    v.backward()
    vc.backward()
    assert torch.equal(big.grad[..., :96], ac.grad) and torch.equal(big.grad[..., 96:], bc.grad)
    lib = _lib.load()
    x = ac.detach().requires_grad_(True)
    n0 = lib.r3dg_launch_count()
    fused(x, bc.detach(), True).backward()
    torch.cuda.synchronize()
    assert lib.r3dg_launch_count() - n0 == 3           # forward tiles + reduction, one backward
    assert torch.equal(x.grad, ac.grad)


def test_rejects_what_the_call_sites_never_pass():
    a = torch.rand(2, 3, 16, 16, device="cuda")
    with pytest.raises(ValueError, match="window_size"):
        fused_ws(a, a, 9)
    with pytest.raises(TypeError, match="float32"):
        fused(a.double(), a.double(), True)
    with pytest.raises(TypeError, match="float32"):
        fused(a.half(), a.half(), True)
    with pytest.raises(ValueError, match="CUDA"):
        fused(a.cpu(), a.cpu(), True)
    with pytest.raises(ValueError, match="shapes differ"):
        fused(a, a[:, :, :15], True)
    with pytest.raises(ValueError, match="size_average=False"):
        fused(a[0], a[0], False)
    x = a.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(fused(x, a.flip(-1), True), x, create_graph=True)
    with pytest.raises(RuntimeError):
        g.sum().backward()


def fused_ws(a, b, window_size):
    from relightable3dgaussian_b200.losses import ssim
    return ssim(a, b, window_size)
