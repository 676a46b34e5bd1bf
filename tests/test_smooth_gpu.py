"""GPU parity of the fused smoothness regularisers (relightable3dgaussian_b200.losses.first_order_edge_aware_loss and
tv_loss) against the reference formula in fp64.  e_kernel is the fused result's error against that truth, e_ref the
error of the IEEE fp32 reference formula (the fixture's fp32 record, or tests/smooth_oracle.py in fp32 on the GPU).
Values pass at |e_kernel| <= max(1e-6 |L|, 4 e_ref), gradients by relative L2 at <= max(2e-6, 4 e_ref).  Where the
truth is exactly 0 (constant data, a 1x1 image, the img gradient on a constant img) the fused result must be exactly
0 too."""
import os

import numpy as np
import pytest
import torch

import smooth_oracle as so
from helpers import GOLDEN, npy, rel_l2

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(GOLDEN, "smooth.npz"))


def fused_edge(d, i):
    from relightable3dgaussian_b200.losses import first_order_edge_aware_loss
    return first_order_edge_aware_loss(d, i)


def fused_tv(x):
    from relightable3dgaussian_b200.losses import tv_loss
    return tv_loss(x)


def run(fn, inputs, need, cot, dtype):
    """(value, [dL/dinput or None ...]) of fn(*inputs) in `dtype`, L = value * cot, gradients only where `need`."""
    xs = [t.detach().to(dtype).requires_grad_(n) for t, n in zip(inputs, need)]
    with so.ieee_convolutions():
        v = fn(*xs)
        (v * cot.to(v)).backward()
    return npy(v), [npy(x.grad) for x in xs]


def check(tag, mine, truth, ref32):
    """mine / truth / ref32: (value, [grads]); a None gradient is not checked.  Returns the ratios e_kernel / e_ref."""
    ek = abs(float(mine[0]) - float(truth[0]))
    er = abs(float(ref32[0]) - float(truth[0]))
    if float(truth[0]) == 0.0:
        assert float(mine[0]) == 0.0, (tag, "value", float(mine[0]))
    assert ek <= max(1e-6 * abs(float(truth[0])), 4 * er), (tag, "value", ek, er)
    ratios = [ek / max(er, 1e-30)]
    for k, (m, t, r) in enumerate(zip(mine[1], truth[1], ref32[1])):
        if m is None:
            continue
        assert m.shape == t.shape and m.dtype == np.float32, (tag, k)
        if not t.any():
            assert not m.any(), (tag, f"grad{k} must be exactly 0", np.abs(m).max())
            ratios.append(0.0)
            continue
        ek, er = rel_l2(m, t), rel_l2(r, t)
        assert ek <= max(2e-6, 4 * er), (tag, f"grad{k}", ek, er)
        ratios.append(ek / max(er, 1e-30))
    print(f"[smooth] {tag:40s} e_kernel/e_ref " + " ".join(f"{x:.2f}" for x in ratios))
    return ratios


@pytest.mark.parametrize("case", so.EDGE_CASES, ids=[c[0] for c in so.EDGE_CASES])
def test_edge_aware_matches_reference_function_golden(case):
    name, kind, Cd, Ci, H, W, seed = case
    d, i, cot = so.smooth_case(kind, Cd, Ci, H, W, seed)
    mine = run(fused_edge, [d.cuda(), i.cuda()], (True, True), cot.cuda(), torch.float32)
    truth = (G[f"edge/{name}/value64"], [G[f"edge/{name}/grad_data64"], G[f"edge/{name}/grad_img64"]])
    ref32 = (G[f"edge/{name}/value32"], [G[f"edge/{name}/grad_data32"], G[f"edge/{name}/grad_img32"]])
    assert mine[0].shape == ()
    check(name, mine, truth, ref32)


@pytest.mark.parametrize("case", so.TV_CASES, ids=[c[0] for c in so.TV_CASES])
def test_tv_matches_reference_function_golden(case):
    name, shape, permuted, seed = case
    x, cot = so.tv_case(shape, permuted, seed)
    x = x.cuda() if not permuted else x.permute(1, 2, 0).cuda().permute(2, 0, 1)     # keep the permuted layout
    assert x.is_contiguous() != permuted
    mine = run(fused_tv, [x], (True,), cot.cuda(), torch.float32)
    check(name, mine, (G[f"tv/{name}/value64"], [G[f"tv/{name}/grad64"]]), (G[f"tv/{name}/value32"], [G[f"tv/{name}/grad32"]]))


SIZES = [(800, 800), (1200, 1600), (1080, 1920)]
PAIRS = [(3, 3, (True, False)), (1, 3, (True, False)), (3, 3, (True, True))]


@pytest.mark.parametrize("kind", ["rendered", "masked"])
@pytest.mark.parametrize("pair", PAIRS, ids=["3x3", "1x3", "3x3_img_grad"])
@pytest.mark.parametrize("size", SIZES, ids=["x".join(map(str, s)) for s in SIZES])
def test_edge_aware_matches_ieee_oracle_at_training_sizes(size, pair, kind):
    Cd, Ci, need = pair
    d, i, cot = so.smooth_case(kind, Cd, Ci, *size, seed=21)
    inputs, cot = [d.cuda(), i.cuda()], cot.cuda()
    truth = run(so.first_order_edge_aware_loss, inputs, need, cot, torch.float64)
    ref32 = run(so.first_order_edge_aware_loss, inputs, need, cot, torch.float32)
    mine = run(fused_edge, inputs, need, cot, torch.float32)
    assert all((g is None) == (not n) for g, n in zip(mine[1], need))
    check(f"{kind} {Cd}x{Ci} {size} need={need}", mine, truth, ref32)


def test_tv_matches_ieee_oracle_at_training_sizes():
    for shape in [(3, 1200, 1600), (3, 256, 512)]:
        x = torch.rand(shape, generator=torch.Generator().manual_seed(5)).cuda()
        cot = torch.tensor(0.7, device="cuda")
        truth, ref32, mine = (run(fn, [x], (True,), cot, dt) for fn, dt in
                              ((so.tv_loss, torch.float64), (so.tv_loss, torch.float32), (fused_tv, torch.float32)))
        check(f"tv {shape}", mine, truth, ref32)


def test_constant_inputs_give_exact_zeros_at_training_size():
    d, i, cot = so.smooth_case("constdata", 3, 3, 1080, 1920, seed=3)
    v, (gd, gi) = run(fused_edge, [d.cuda(), i.cuda()], (True, True), cot.cuda(), torch.float32)
    assert float(v) == 0.0 and not gd.any() and not gi.any()
    d, i, cot = so.smooth_case("constimg", 1, 3, 1080, 1920, seed=4)
    _, (gd, gi) = run(fused_edge, [d.cuda(), i.cuda()], (True, True), cot.cuda(), torch.float32)
    assert gd.any() and not gi.any()
    x = torch.full((2, 3, 64, 80), 0.25, device="cuda", requires_grad=True)
    fused_tv(x).backward()
    assert not x.grad.any()


def test_deterministic():
    d, i, cot = so.smooth_case("masked", 1, 3, 1200, 1600, seed=5)
    r1, r2 = (run(fused_edge, [d.cuda(), i.cuda()], (True, True), cot.cuda(), torch.float32) for _ in range(2))
    assert np.array_equal(r1[0], r2[0]) and all(np.array_equal(a, b) for a, b in zip(r1[1], r2[1]))
    x = torch.rand(3, 1200, 1600, device="cuda")
    t1, t2 = (run(fused_tv, [x], (True,), cot.cuda(), torch.float32) for _ in range(2))
    assert np.array_equal(t1[0], t2[0]) and np.array_equal(t1[1][0], t2[1][0])


def test_launch_counts_and_requested_gradients():
    """Forward: tiles + reduction; backward: one launch whichever gradients are requested."""
    from relightable3dgaussian_b200 import _lib
    lib = _lib.load()
    d, i, _ = so.smooth_case("rendered", 3, 1, 64, 96, seed=6)
    d, i = d.cuda(), i.cuda()
    for need in ((True, False), (False, True), (True, True)):
        a, b = d.clone().requires_grad_(need[0]), i.clone().requires_grad_(need[1])
        torch.cuda.synchronize()
        n0 = lib.r3dg_launch_count()
        fused_edge(a, b).backward()
        torch.cuda.synchronize()
        assert lib.r3dg_launch_count() - n0 == 3, need
        assert (a.grad is not None) == need[0] and (b.grad is not None) == need[1]
    x = torch.rand(3, 40, 50, device="cuda", requires_grad=True)
    n0 = lib.r3dg_launch_count()
    fused_tv(x).backward()
    torch.cuda.synchronize()
    assert lib.r3dg_launch_count() - n0 == 3
    n0 = lib.r3dg_launch_count()
    with torch.no_grad():
        fused_edge(d, i), fused_tv(x)
    assert lib.r3dg_launch_count() - n0 == 4


def test_non_contiguous_views_are_bit_identical_to_contiguous_copies():
    big = torch.rand(3, 80, 2 * 96, device="cuda", requires_grad=True)
    a, b = big.split(96, dim=-1)
    b = b[1:2]                                          # a 1-channel img, as roughness-like broadcasting
    assert not a.is_contiguous() and not b.is_contiguous()
    ac, bc = a.detach().contiguous().requires_grad_(True), b.detach().contiguous().requires_grad_(True)
    v, vc = fused_edge(a, b), fused_edge(ac, bc)
    assert torch.equal(v, vc)
    v.backward()
    vc.backward()
    assert torch.equal(big.grad[..., :96], ac.grad) and torch.equal(big.grad[1:2, :, 96:], bc.grad)
    env = torch.randn(1, 32, 64, 3, device="cuda", requires_grad=True)
    x = env[0].permute(2, 0, 1)                         # gaussian_renderer/neilf.py:306
    xc = x.detach().contiguous().requires_grad_(True)
    t, tc = fused_tv(x), fused_tv(xc)
    assert torch.equal(t, tc)
    t.backward()
    tc.backward()
    assert torch.equal(env.grad[0].permute(2, 0, 1), xc.grad)


def test_stage2_regularizer_mix_matches_oracle():
    """EA(base m, gt) + 0.5 EA(rough m, gt) + EA(diffuse m, normal) + 0.01 tv(softplus(env)[0].permute(2, 0, 1)),
    the regularisers gaussian_renderer/neilf.py:284-306 add, with gradients to every rendered attribute and env."""
    H, W = 400, 600
    g = torch.Generator().manual_seed(8)
    m, _ = so._mask(H, W, g)
    base, rough, diffuse, gt = (so._rendered(c, H, W, g) for c in (3, 1, 3, 3))
    normal = torch.nn.functional.normalize(so._rendered(3, H, W, g) * 2 - 1, dim=0)
    env = torch.randn(1, 64, 128, 3, generator=g)
    leaves = [t.cuda() for t in (base, rough, diffuse, normal, env)]
    m, gt = m.cuda(), gt.cuda()

    def mix(ea, tv):
        def f(b, r, d, n, e):
            return (ea(b * m, gt) + 0.5 * ea(r * m, gt) + ea(d * m, n)
                    + 0.01 * tv(torch.nn.functional.softplus(e)[0].permute(2, 0, 1)))
        return f

    need = (True,) * 5
    cot = torch.tensor(1.0, device="cuda")
    mine = run(mix(fused_edge, fused_tv), leaves, need, cot, torch.float32)
    truth = run(mix(so.first_order_edge_aware_loss, so.tv_loss), leaves, need, cot, torch.float64)
    ref32 = run(mix(so.first_order_edge_aware_loss, so.tv_loss), leaves, need, cot, torch.float32)
    ratios = check("stage-2 mix", mine, truth, ref32)
    assert len(ratios) == 6 and all(gr.any() for gr in mine[1])


def test_rejects_what_the_call_sites_never_pass():
    a = torch.rand(3, 16, 16, device="cuda")
    for bad in (a.double(), a.half()):
        with pytest.raises(TypeError, match="float32"):
            fused_edge(bad, a)
        with pytest.raises(TypeError, match="float32"):
            fused_edge(a, bad)
        with pytest.raises(TypeError, match="float32"):
            fused_tv(bad)
    with pytest.raises(ValueError, match="CUDA"):
        fused_edge(a.cpu(), a)
    with pytest.raises(ValueError, match="CUDA"):
        fused_edge(a, a.cpu())
    with pytest.raises(ValueError, match="CUDA"):
        fused_tv(a.cpu())
    for bad in (a[0], a[None]):
        with pytest.raises(ValueError, match=r"\[C,H,W\]"):
            fused_edge(bad, a)
        with pytest.raises(ValueError, match=r"\[C,H,W\]"):
            fused_edge(a, bad)
    with pytest.raises(ValueError, match="sizes differ"):
        fused_edge(a, a[:, :15])
    with pytest.raises(ValueError, match="sizes differ"):
        fused_edge(a[:, :, :15], a)
    with pytest.raises(ValueError, match="broadcast"):
        fused_edge(a[:2], a)
    with pytest.raises(ValueError, match="broadcast"):
        fused_edge(torch.rand(4, 16, 16, device="cuda"), a)
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="devices"):
            fused_edge(a, a.to("cuda:1"))
    with pytest.raises(ValueError, match=r"\[\.\.\., H, W\]"):
        fused_tv(a[0, 0])
    for bad in (a[:, :1], a[:, :, :1], a[0, :1]):
        with pytest.raises(ValueError, match="at least 2"):
            fused_tv(bad)
    x = a.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad(fused_edge(x, a.flip(-1)), x, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()
    (gx,) = torch.autograd.grad(fused_tv(x), x, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()
