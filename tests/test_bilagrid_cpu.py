"""Bilateral-grid slice without a GPU: the fp64 numpy restatement (tests/bilagrid_oracle.py) against
F.grid_sample + autograd in fp64, the grids' TV term against an explicit sum, and the argument checks of the C ABI and
of bilagrid.slice, none of which may launch anything."""
import ctypes

import numpy as np
import pytest
import torch

import bilagrid_oracle as bo
from relightable3dgaussian_b200 import _lib, bilagrid


def _torch64(grids, rgb, ids, dout):
    g = torch.tensor(grids, dtype=torch.float64, requires_grad=True)
    x = torch.tensor(rgb, dtype=torch.float64, requires_grad=True)
    out = bo.torch_slice(g, x, ids)
    out.backward(torch.tensor(dout, dtype=torch.float64))
    return out.detach().numpy(), x.grad.numpy(), g.grad.numpy()


# (name, G, ids, H, W, L, GY, GX, luma range)
CASES = [
    ("in_range", 2, [1], 20, 28, 8, 16, 16, (0.02, 0.98)),
    ("below_zero", 1, [0], 12, 17, 8, 6, 5, (-0.6, -0.05)),
    ("above_one", 1, [0], 13, 11, 5, 4, 7, (1.05, 1.7)),
    ("straddling", 2, [0, 1], 16, 16, 6, 5, 5, (-0.3, 1.3)),
    ("repeated_ids", 3, [2, 0, 2, 2], 10, 14, 4, 3, 6, (0.0, 1.0)),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_matches_grid_sample_autograd_fp64(case):
    _, G, ids, H, W, L, GY, GX, (lo, hi) = case
    grids, rgb = bo.random_case(G, len(ids), H, W, L, GY, GX, seed=len(ids) + H, luma_lo=lo, luma_hi=hi, noise=0.3)
    dout = np.random.default_rng(7).standard_normal(rgb.shape)
    out, drgb, dgrids = _torch64(grids, rgb, ids, dout)
    out64 = bo.slice64(grids, rgb, ids)
    drgb64, dgrids64, iz = bo.grads64(grids, rgb, ids, dout)
    np.testing.assert_allclose(out64, out, rtol=0, atol=1e-12)
    np.testing.assert_allclose(dgrids64, dgrids, rtol=0, atol=1e-11 * max(np.abs(dgrids).max(), 1))
    keep = ~bo.near_node_mask(iz, L)[:, None]
    assert keep.mean() > 0.99
    np.testing.assert_allclose(np.where(keep, drgb64, 0), np.where(keep, drgb, 0), rtol=0, atol=1e-11)
    if hi < 0 or lo > 1:           # the whole image beyond the border: no luma term, dL/drgb = A^T dL/dout
        A = np.stack([bo.affine(grids[g].astype(np.float64), rgb[n].astype(np.float64)) for n, g in enumerate(ids)])
        A = A.reshape(len(ids), 3, 4, H, W)
        np.testing.assert_allclose(drgb64, np.einsum("ncjhw,nchw->njhw", A[:, :, :3], dout), rtol=0, atol=1e-12)
    if len(set(ids)) < len(ids):   # repeated ids sum: each view's gradient alone, added up
        parts = [bo.grads64(grids, rgb[n:n + 1], [g], dout[n:n + 1])[1] for n, g in enumerate(ids)]
        np.testing.assert_allclose(dgrids64, sum(parts), rtol=0, atol=1e-12)


def test_identity_and_constant_grids():
    """The identity grid returns its input and a constant grid applies its one affine matrix, in the oracle and in the
    torch formulation (fp64, which weight products rather than nested lerps: to rounding)."""
    grids, rgb = bo.random_case(1, 1, 9, 13, 4, 3, 5, seed=3, luma_lo=-0.2, luma_hi=1.2, noise=0.0)
    np.testing.assert_allclose(bo.slice64(grids, rgb, [0]), rgb.astype(np.float64), rtol=0, atol=1e-15)
    M = np.random.default_rng(1).standard_normal(12)
    const = np.broadcast_to(M.reshape(1, 12, 1, 1, 1), grids.shape).copy()
    want = np.einsum("cj,njhw->nchw", M.reshape(3, 4)[:, :3], rgb.astype(np.float64)) + M.reshape(3, 4)[:, 3, None, None]
    np.testing.assert_allclose(bo.slice64(const, rgb, [0]), want, rtol=0, atol=1e-13)
    out = bo.torch_slice(torch.tensor(const), torch.tensor(rgb, dtype=torch.float64), [0]).numpy()
    np.testing.assert_allclose(out, want, rtol=0, atol=1e-13)


def test_tv_loss_is_the_sum_of_mean_squared_forward_differences():
    m = bilagrid.BilateralGrid(3, grid_X=5, grid_Y=4, grid_W=3)
    assert m.grids.shape == (3, 12, 3, 4, 5)
    np.testing.assert_array_equal(m.grids.detach().numpy()[:, :, 1, 2, 3], np.tile(bo.IDENTITY, (3, 1)))
    assert m.tv_loss().item() == 0.0
    with torch.no_grad():
        m.grids.add_(torch.from_numpy(np.random.default_rng(0).standard_normal(m.grids.shape).astype(np.float32)))
    g = m.grids.detach().double().numpy()
    want = 0.0
    for axis in (2, 3, 4):
        n = g.shape[axis]
        total, count = 0.0, 0
        for i in range(n - 1):
            d = np.take(g, i + 1, axis=axis) - np.take(g, i, axis=axis)
            total += float((d * d).sum())
            count += d.size
        want += total / count
    tv = m.tv_loss()
    assert tv.dtype == torch.float32 and tv.dim() == 0
    assert abs(tv.item() - want) <= 1e-5 * want
    tv.backward()
    assert m.grids.grad is not None and m.grids.grad.shape == m.grids.shape


P = ctypes.c_void_p(256)          # never dereferenced: every call below fails its checks first


def test_abi_rejects_bad_arguments_before_launching():
    lib = _lib.load()
    n0 = lib.r3dg_launch_count()
    good = (2, 3, 64, 80, 16, 16, 8)       # G, N, H, W, GX, GY, L
    tmp = lib.r3dg_bilagrid_tmp_bytes(*good)
    assert tmp > 0 and tmp % 256 == 0 and lib.r3dg_bilagrid_tmp_bytes(2, 6, 64, 80, 16, 16, 8) > tmp
    fwd = lambda shape, *ptrs: lib.r3dg_bilagrid_forward(*shape, *ptrs, None)
    bwd = lambda shape, *ptrs, nbytes=tmp: lib.r3dg_bilagrid_backward(*shape, *ptrs, nbytes, None)
    bad_shapes = [(0, 3, 64, 80, 16, 16, 8), (2, 0, 64, 80, 16, 16, 8), (2, 3, 0, 80, 16, 16, 8),
                  (2, 3, 64, -1, 16, 16, 8), (2, 3, 64, 80, 1, 16, 8), (2, 3, 64, 80, 16, 1, 8),
                  (2, 3, 64, 80, 16, 16, 1), (2, 3, 64, 80, 16, 16, 0)]
    unsupported = [(2, 65536, 64, 80, 16, 16, 8), (2, 3, 64, 80, 16, 16, 17), (2, 3, 64, 80, 1025, 16, 8),
                   (2, 3, 1 << 16, 1 << 15, 16, 16, 8), (1 << 14, 3, 64, 80, 64, 64, 16),
                   (2, 3, 16, 16, 16, 16, 8),          # the sub-grid of one tile: 16 x 16 x 8 nodes
                   (2, 3, 51, 51, 16, 16, 8)]          # 12 x 12 x 8 > 1024
    for shape, code in [(s, -10001) for s in bad_shapes] + [(s, -10002) for s in unsupported]:
        assert lib.r3dg_bilagrid_tmp_bytes(*shape) == 0, shape
        assert fwd(shape, P, P, P, P) == code, shape
        assert bwd(shape, P, P, P, P, P, P, P, nbytes=1 << 30) == code, shape
    for k in range(4):                                 # a NULL in each pointer the forward needs
        ptrs = [P] * 4
        ptrs[k] = None
        assert fwd(good, *ptrs) == -10001, k
    for k in range(4):                                 # grids, ids, rgb, dL_dout
        ptrs = [P] * 7
        ptrs[k] = None
        assert bwd(good, *ptrs) == -10001, k
    assert bwd(good, P, P, P, P, None, None, P) == -10001          # no output asked for
    assert bwd(good, P, P, P, P, P, P, None) == -10001             # dL_dgrids without a workspace
    assert bwd(good, P, P, P, P, P, P, P, nbytes=tmp - 1) == -10001
    assert lib.r3dg_launch_count() == n0
    # the smallest images gsplat's default grid fits, as the header states
    assert lib.r3dg_bilagrid_tmp_bytes(1, 1, 52, 52, 16, 16, 8) > 0
    assert lib.r3dg_bilagrid_tmp_bytes(1, 1, 51, 52, 16, 16, 8) == 0


def test_slice_rejects_bad_ids_and_dtypes_on_the_host():
    lib = _lib.load()
    n0 = lib.r3dg_launch_count()
    grids = bilagrid.BilateralGrid(3, 4, 4, 2).grids.detach()
    rgb = torch.rand(2, 3, 8, 8)
    for ids, exc in (([0, 3], ValueError), ([-1, 0], ValueError), ([0], ValueError), ([0, 1, 2], ValueError),
                     (torch.tensor([0.0, 1.0]), TypeError), ([0, 1.0], TypeError), ([True, 0], TypeError),
                     (torch.tensor([0, 5]), ValueError), (7, ValueError)):
        with pytest.raises(exc):
            bilagrid.slice(grids, rgb, ids)
    with pytest.raises(TypeError, match="float32"):
        bilagrid.slice(grids.double(), rgb, [0, 1])
    with pytest.raises(TypeError, match="float32"):
        bilagrid.slice(grids, rgb.half(), [0, 1])
    with pytest.raises(ValueError, match=r"\[3,H,W\]"):
        bilagrid.slice(grids, torch.rand(2, 4, 8, 8), [0, 1])
    with pytest.raises(ValueError, match="GY,GX"):
        bilagrid.slice(grids[:, :6], rgb, [0, 1])
    with pytest.raises(ValueError, match="CUDA"):
        bilagrid.slice(grids, rgb, torch.tensor([0, 2]))    # valid ids: the device check comes next
    assert bilagrid._host_ids(torch.tensor([[2], [0]], dtype=torch.int16), 2, 3) == [2, 0]
    assert bilagrid._host_ids(np.int64(1), 1, 3) == [1]
    assert lib.r3dg_launch_count() == n0
