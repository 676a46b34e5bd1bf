"""SSIM without a GPU: the PyTorch restatement (tests/ssim_oracle.py) against the outputs and autograd
gradients of the reference's own function bodies (tests/golden/ssim.npz), the window the kernels
use, argument checks of the C ABI, and install() / uninstall()."""
import ctypes
import os
import re
import types

import numpy as np
import pytest
import torch

import ssim_oracle as oss
from helpers import GOLDEN, ROOT, rel_l2
from relightable3dgaussian_b200 import _lib

G = np.load(os.path.join(GOLDEN, "ssim.npz"))


@pytest.mark.parametrize("case", oss.GOLDEN_CASES, ids=[c[0] for c in oss.GOLDEN_CASES])
def test_oracle_matches_reference_function_golden(case):
    """fp64 agrees to 1e-12.  In fp32 the oracle runs the reference's op sequence, so on the machine
    that wrote the fixture the results are bit-identical; oneDNN picks its CPU convolution kernels by
    instruction set, so a few ulp are allowed elsewhere."""
    name, kind, shape, size_average, seed = case
    a, b, cot = oss.ssim_case(kind, shape, seed)
    fn = lambda x, y, sa: oss.ssim(x, y, size_average=sa)
    v, g1, g2 = oss.value_and_grads(fn, a, b, cot, size_average, torch.float64)
    np.testing.assert_allclose(v.numpy(), G[f"{name}/value64"], rtol=0, atol=1e-12)
    for k, g in (("grad1", g1), ("grad2", g2)):
        ref = G[f"{name}/{k}_64"]
        assert np.abs(g.numpy() - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-3), k
    v, g1, g2 = oss.value_and_grads(fn, a, b, cot, size_average, torch.float32)
    np.testing.assert_allclose(v.numpy(), G[f"{name}/value32"], rtol=1e-6, atol=0)
    for k, g in (("grad1", g1), ("grad2", g2)):
        ref = G[f"{name}/{k}_32"]
        assert np.abs(g.numpy() - ref).max() <= 1e-6 * np.abs(ref).max() + 1e-12, k
    assert v.shape == (() if size_average else (shape[0],))


def test_window_is_the_references():
    """gaussian(11, 1.5) of loss_utils.py:20-22 (exp in double, float32, / float32 sum): the oracle's and the
    kernels' constant table (csrc/ssim.cu) against the reference's own result, and the kernels' correction of
    the separable window's total weight to that of the reference's float32 2-D window."""
    ref = G["window1d"]
    assert ref.dtype == np.float32 and ref.shape == (11,)
    np.testing.assert_allclose(oss.gaussian(11, 1.5).numpy(), ref, rtol=2.5e-7, atol=0)
    src = open(os.path.join(ROOT, "relightable3dgaussian_b200", "csrc", "ssim.cu")).read()
    table = re.search(r"__constant__ float kW\[11\] = \{(.*?)\};", src, re.S).group(1)
    kernel = np.array([float.fromhex(t.strip().rstrip("f")) for t in table.split(",")], np.float32)
    assert np.array_equal(kernel, ref), (kernel, ref)
    assert np.array_equal(kernel, kernel[::-1])          # symmetric: the transposed blur is the same blur
    w = ref.astype(np.float64)
    window_2d = np.float32(w[:, None] * w[None, :])      # create_window: the float32 mm of [11,1] x [1,11]
    gain_err = np.float32(window_2d.astype(np.float64).sum() / w.sum() ** 2 - 1)
    stated = float.fromhex(re.search(r"constexpr float kGainErr = (\S+)f;", src).group(1))
    assert np.float32(stated) == gain_err, (stated, gain_err)


def test_abi_rejects_bad_arguments_before_launching():
    lib = _lib.load()
    n0 = lib.r3dg_launch_count()
    tmp = lib.r3dg_ssim_tmp_bytes(2, 3, 40, 50)
    assert tmp > 0 and tmp % 256 == 0 and lib.r3dg_ssim_tmp_bytes(2, 3, 400, 500) > tmp
    p = ctypes.c_void_p(256)                 # never dereferenced: every call below fails its checks first
    for N, C, H, W in ((0, 3, 8, 8), (1, 0, 8, 8), (1, 3, 0, 8), (1, 3, 8, 0), (-1, 3, 8, 8), (1, 3, 8, -2)):
        assert lib.r3dg_ssim_tmp_bytes(N, C, H, W) == 0
        assert lib.r3dg_ssim_forward(N, C, H, W, p, p, 1, p, p, 1 << 20, None) == -10001
        assert lib.r3dg_ssim_backward(N, C, H, W, p, p, 1, p, p, None) == -10001
    for k in range(4):                         # a NULL in each pointer argument
        ptrs = [p] * 4
        ptrs[k] = None
        assert lib.r3dg_ssim_forward(2, 3, 40, 50, ptrs[0], ptrs[1], 0, ptrs[2], ptrs[3], tmp, None) == -10001
        assert lib.r3dg_ssim_backward(2, 3, 40, 50, *ptrs[:2], 0, *ptrs[2:], None) == -10001
    assert lib.r3dg_ssim_forward(2, 3, 40, 50, p, p, 0, p, p, tmp - 1, None) == -10001
    assert lib.r3dg_ssim_forward(65536, 1, 8, 8, p, p, 0, p, p, 1 << 30, None) == -10002
    assert lib.r3dg_ssim_backward(1, 1, 1 << 16, 1 << 15, p, p, 0, p, p, None) == -10002
    assert lib.r3dg_launch_count() == n0


def test_install_rebinds_and_uninstall_restores():
    from relightable3dgaussian_b200 import losses
    orig = object()
    mods = [types.ModuleType(n) for n in ("stub_loss_utils", "stub_render", "stub_neilf")]
    for m in mods:
        m.ssim = orig
    try:
        assert losses.install(*mods) == mods
        assert all(m.ssim is losses.ssim for m in mods)
    finally:
        losses.uninstall()
    assert all(m.ssim is orig for m in mods)
    assert losses.DEFAULT_MODULES == ("utils.loss_utils", "gaussian_renderer.render", "gaussian_renderer.neilf")


def test_rejects_what_the_call_sites_never_pass_without_a_gpu():
    from relightable3dgaussian_b200.losses import ssim
    a = torch.rand(3, 8, 8)
    with pytest.raises(ValueError, match="window_size"):
        ssim(a, a, window_size=7)
    with pytest.raises(ValueError, match="CUDA"):
        ssim(a, a)
